"""The occupancy-grid update (csrc/grid_update.cu and DensityGridSampler.update_density_grid) against the oracle and float64 at
training sizes.

  * sample generation: G3 and 3 G3 draws (lego's and fox's step-0..255 update) and their quarters (from step 256 on), both thresholds,
    at ema steps 0, 1, the first step where step * n passes 2^32, and a large int32 step -- indices and positions bit for bit (that the
    32-bit wrap cannot change an index is shown in test_march_bound_cpu.py);
  * splat: fp16 (what density_fwd returns, the training dtype) and fp32 on millions of colliding indices, each cell against the float64
    max of exp(x) * fl(sqrt(3))/1024 with a per-entry bound (__expf's documented 2 + floor(|1.173 x|) ulp, then the product's rounding);
    fp16 edge inputs ±0, ±inf, ±65504 and products below 2^-126.  The kernel evaluates __expf without flush-to-zero (ex2.approx.f32 with
    the subnormal range rescaled, and an IEEE multiply): a sample with x in about [-103, -83] leaves a positive subnormal in its cell,
    which is occupied when the threshold is a mean of 0 -- asserted below;
  * ema bit for bit at 5 cascades; the mean of ngp_grid_update_bitfield bit for bit against march_ref.mean_f32 (the kernels' fixed
    order restated) and within march_ref.mean_bound of the float64 mean, above and below 0.01; the bitfield bit for bit given the kernel's mean (every max-pool level), and equal to the fp64-mean bitfield except in cells
    within the bound of the threshold;
  * DensityGridSampler.update_density_grid on a Runner (lego stand-in, fox config) at step 0 and across 255 -> 256, against the oracle
    chain fed with the sampler's own fp16 densities: positions, rng, ema step, the cleared density_grid_tmp, grid, mean and bitfield."""
import numpy as np
import pytest
import torch

import march_ref as M
import oracle_lib as ol

pytestmark = pytest.mark.gpu

G3 = M.G3
MIN_OPT = 0.01                                                           # NERF_MIN_OPTICAL_THICKNESS


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def npy(t):
    return t.detach().cpu().numpy()


def _grid(seed=0, cascades=5):
    """-1 (never seen), 0, values either side of 0.01 and of a small mean: what a grid holds a few updates into training."""
    rng = np.random.default_rng(seed)
    n = G3 * cascades
    u = rng.random(n)
    g = np.where(u < 0.2, -1.0, np.where(u < 0.5, 0.0, rng.random(n) * 0.02)).astype(np.float32)
    return g


def _first_wrap(n):
    return -(-(1 << 32) // n)                                            # smallest step with step * n >= 2^32


CASES = [(n, s) for n in (G3, 3 * G3, G3 // 4, 3 * G3 // 4) for s in (0, 1, _first_wrap(n), 2 ** 31 - 1)]


@pytest.mark.parametrize("thresh", [-0.01, MIN_OPT])
@pytest.mark.parametrize("n,step", CASES)
def test_generate_samples(ops, n, step, thresh):
    n_cascades = 3 if n % 3 == 0 else 1                                  # fox (aabb_scale 4) draws over 3 cascades, lego over 1
    aabb = (-1.5, 2.5) if n_cascades == 3 else (0.0, 1.0)
    g = _grid(n + step)
    si = ol.pcg32_advance(ol.pcg32_seed(), step * 7919)
    pos, idx = ops.grid_generate_samples(n, si, torch.tensor([step], dtype=torch.int32, device="cuda"), aabb, cu(g), n_cascades, thresh)
    pr, ir = ol.generate_grid_samples(n, si, step, aabb, g, n_cascades, thresh)
    assert np.array_equal(npy(idx).view(np.uint32), ir)
    assert np.array_equal(npy(pos).view(np.uint32), pr.view(np.uint32))


EDGE16 = np.array([0.0, -0.0, np.inf, -np.inf, 65504.0, -65504.0, -83.0, -88.0, -90.0, -95.0, -104.0, -110.0, 11.0, -11.0], np.float16)


def _splat_check(got, idx, x):
    """every cell: max over its samples of ref - bound <= got <= max of ref + bound; cells no sample hit stay 0"""
    ref, b = M.splat_ref(x.astype(np.float64))
    lo = np.where(np.isinf(ref), np.inf, ref - b)
    hi = ref + b
    clo = np.full(got.size, -np.inf)
    chi = np.full(got.size, -np.inf)
    np.maximum.at(clo, idx, lo)
    np.maximum.at(chi, idx, hi)
    hit = chi > -np.inf
    g = got.astype(np.float64)
    assert (g[~hit] == 0).all()
    ok = (g[hit] >= np.maximum(clo[hit], 0)) & (g[hit] <= chi[hit])
    assert ok.all(), f"{int((~ok).sum())} cells outside the bound, e.g. {np.flatnonzero(hit)[~ok][:4].tolist()}"
    return int(hit.sum())


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_splat_against_float64(ops, dtype):
    n = 3 * G3
    si = ol.pcg32_seed()
    _, idx = ops.grid_generate_samples(n, si, torch.tensor([5], dtype=torch.int32, device="cuda"), (-1.5, 2.5), cu(_grid(1)), 3, MIN_OPT)
    rng = np.random.default_rng(2)
    x = (rng.standard_normal(n) * 4).astype(dtype)
    x[rng.integers(0, n, 4000)] = np.tile(EDGE16, 4000 // EDGE16.size + 1)[:4000].astype(dtype)
    tmp = torch.zeros(G3 * 5, dtype=torch.float32, device="cuda")
    ops.grid_splat(idx, cu(x), tmp)
    ii = npy(idx).view(np.uint32)
    hit = _splat_check(npy(tmp), ii, x)
    print(f"[grid] splat {np.dtype(dtype).name}: {n} samples into {hit} cells")


def test_splat_fp16_edges_no_flush_to_zero(ops):
    x = EDGE16
    idx = (np.arange(x.size, dtype=np.uint32) * 97).astype(np.int32)     # one sample a cell
    tmp = torch.zeros(G3 * 5, dtype=torch.float32, device="cuda")
    ops.grid_splat(cu(idx), cu(x), tmp)
    got = npy(tmp)[idx.view(np.uint32)]
    _splat_check(npy(tmp), idx.view(np.uint32), x)
    assert got[0] == got[1] and abs(got[0] - M.THICK) <= 6 * M.U * M.THICK
    assert np.isinf(got[2]) and np.isinf(got[4]) and got[3] == 0 and got[5] == 0
    sub = got[6:10]                                                      # x = -83, -88, -90, -95: positive subnormal products, not flushed
    assert (sub > 0).all() and (sub < 2.0 ** -126).all(), sub
    assert got[11] == 0                                                  # x = -110: exp(x) * c below half the smallest subnormal
    # with only such cells the mean is at most the smallest subnormal (each addend sub / 2^21 rounds to 0 or 2^-149), and so is the
    # threshold min(0.01, mean): those cells are occupied
    grid = np.zeros(G3 * 5, np.float32)
    grid[idx[6:10]] = sub
    mean = torch.zeros(1, dtype=torch.float32, device="cuda")
    bits = torch.zeros(G3 * 5 // 8, dtype=torch.uint8, device="cuda")
    ops.grid_update_bitfield(cu(grid), mean, bits, 5)
    b = npy(bits)
    m = float(mean.item())
    assert m <= 2.0 ** -149 < sub.min() and np.float32(m) == M.mean_f32(grid)
    assert np.array_equal(b, ol.update_bitfield(grid, m, 5))
    assert all(b[i // 8] >> (i % 8) & 1 for i in idx[6:10])
    assert int(np.unpackbits(b[:G3 // 8]).sum()) == 4


def test_ema_5_cascades(ops):
    rng = np.random.default_rng(4)
    g = _grid(4)
    tmp = np.where(rng.random(G3 * 5) < 0.5, rng.random(G3 * 5) * 0.03, 0).astype(np.float32)
    gd = cu(g)
    ops.grid_ema(gd, cu(tmp), 0.95)
    gr = g.copy()
    ol.ema(gr, tmp, 0.95)
    assert np.array_equal(npy(gd).view(np.uint32), gr.view(np.uint32))


def _mean_grids():
    rng = np.random.default_rng(5)
    yield "above 0.01", (_grid(6) * 3).astype(np.float32)
    yield "below 0.01", (_grid(7) * 0.3).astype(np.float32)
    yield "const 0.0051", np.full(G3 * 5, np.float32(0.0051), np.float32)
    yield "const 0.011", np.full(G3 * 5, np.float32(0.011), np.float32)
    yield "sparse", np.where(rng.random(G3 * 5) < 0.05, rng.random(G3 * 5), -1).astype(np.float32)


@pytest.mark.parametrize("case", range(5))
def test_mean_and_bitfield(ops, case):
    name, g = list(_mean_grids())[case]
    mean = torch.zeros(1, dtype=torch.float32, device="cuda")
    bits = torch.zeros(G3 * 5 // 8, dtype=torch.uint8, device="cuda")
    ops.grid_update_bitfield(cu(g), mean, bits, 5)
    m = float(mean.item())
    s, _ = M.mean_f64(g)
    bound = M.mean_bound(g)
    assert abs(m - s) <= bound, f"{name}: |{m} - {s}| > {bound}"
    assert np.float32(m).view(np.uint32) == M.mean_f32(g).view(np.uint32)    # the fixed order of the two kernels, bit for bit
    b = npy(bits)
    assert np.array_equal(b, ol.update_bitfield(g, m, 5))                   # every max-pool level, given the kernel's mean
    # against the fp64 mean: the cells thresholded differently are all within the mean's bound of the threshold min(0.01, mean)
    th32 = np.float32(0.01) if np.float32(0.01) < np.float32(m) else np.float32(m)
    th64 = min(float(np.float32(0.01)), s)
    flip = (g > th32) != (g.astype(np.float64) > th64)
    near = np.abs(g.astype(np.float64) - th64) <= bound
    assert not (flip & ~near).any()
    print(f"[grid] mean {name}: {m:.9g} vs {s:.9g} (bound {bound:.3g}); {int(near.sum())} cells may flip, {int(flip.sum())} did")
    if not name.startswith("const"):
        assert near.sum() <= 1000


# ---------------------------------------------------------------------------------------------------- the sampler's update
def _runner(style):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**(lego_cfg if style == "lego" else fox_cfg)(fp16=True, synthetic=True, seed=1))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 8
    cfg.dataset.train.H = cfg.dataset.train.W = 160
    cfg.dataset.val = None
    return Runner()


@pytest.mark.parametrize("style", ["lego", "fox"])
def test_sampler_update_against_oracle_chain(ops, style):
    r = _runner(style)
    s = r.sampler
    n_c = s.max_cascade + 1
    assert n_c == (1 if style == "lego" else 3) and s.NERF_CASCADES == 5
    seen = []
    density = s.model.density

    def spy(pos):
        out = density(pos)
        seen.append((pos.detach().clone(), out.detach().clone()))
        return out
    s.model.density = spy
    ds = s.dataset
    for step in (0, 255, 256):
        s.cfg.m_training_step = step
        grid0 = npy(s.density_grid).copy()
        rng0 = s.rng.copy()
        ema0 = int(s.density_grid_ema_step.item())
        s.density_grid_tmp.fill_(7.0)                                    # must be cleared before the splat
        seen.clear()
        s.update_density_grid()
        torch.cuda.synchronize()
        assert ops.lib.load().ngp_debug_timeout_flag() == 0
        if step == 0:
            g = np.zeros(G3 * 5, np.float32)
            ol.oracle().orc_set_fma_mode(0)
            ol.mark_untrained(g, npy(ds.focal_lengths), npy(ds.transforms_gpu), ds.resolution)
            ol.oracle().orc_set_fma_mode(1)
        else:
            g = grid0
        draws = [(G3 * n_c, -0.01)] if step < 256 else [(G3 * n_c // 4, -0.01), (G3 * n_c // 4, MIN_OPT)]
        rng = rng0.copy()
        pos_r, idx_r = [], []
        for n, th in draws:
            p, i = ol.generate_grid_samples(n, rng, ema0, s.aabb_range, g, n_c, th)
            ol.pcg32_advance(rng)
            pos_r.append(p)
            idx_r.append(i)
        pos_r, idx_r = np.concatenate(pos_r), np.concatenate(idx_r)
        pos_g = np.concatenate([npy(p) for p, _ in seen])
        x = np.concatenate([npy(o).reshape(-1) for _, o in seen])
        assert x.dtype == np.float16 and x.size == idx_r.size
        assert np.array_equal(pos_g.view(np.uint32), pos_r.view(np.uint32))
        assert np.array_equal(s.rng, rng)
        assert int(s.density_grid_ema_step.item()) == ema0 + 1
        tmp = npy(s.density_grid_tmp)
        _splat_check(tmp, idx_r, x)                                     # also: no cell kept the 7.0 written before the update
        # ema is monotone in the splatted value: the grid lies between the ema of the lower and of the upper splat bound
        ref, b = M.splat_ref(x.astype(np.float64))
        lo_c, hi_c = np.zeros(G3 * 5), np.zeros(G3 * 5)
        np.maximum.at(lo_c, idx_r, np.maximum(ref - b, 0))
        np.maximum.at(hi_c, idx_r, ref + b)
        dec = (g * np.float32(0.95)).astype(np.float64)
        got = npy(s.density_grid).astype(np.float64)
        keep = g < 0
        assert np.array_equal(got[keep], g[keep].astype(np.float64))
        assert ((got[~keep] >= np.maximum(dec, lo_c)[~keep]) & (got[~keep] <= np.maximum(dec, hi_c)[~keep])).all()
        m = float(s.density_grid_mean.item())
        gg = npy(s.density_grid)
        assert abs(m - M.mean_f64(gg)[0]) <= M.mean_bound(gg)
        assert np.float32(m).view(np.uint32) == M.mean_f32(gg).view(np.uint32)
        assert np.array_equal(npy(s.density_grid_bitfield), ol.update_bitfield(gg, m, 5))
        print(f"[grid] {style} update at step {step}: {x.size} samples, mean {m:.6g}")
