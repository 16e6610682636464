"""The training march (ngp_march) and compaction (ngp_compact) against the oracle (oracle/ngp_oracle.c, fma_mode 1) at training sizes,
bit for bit: counters, numsteps (counts and ray-ordered bases), ray indices and every emitted row.

Rays are camera rays of the lego stand-in (unit box, const_dt) and of the fox capture (tests/golden/fox_small: aabb_scale 4, cone
stepping) made by ops.raygen, plus rays that start inside the box with near = 0.  Ray counts straddle the 1024 threads of the
single-CTA scans (1023 / 1024 / 1025: per = 1 or 2 rays a thread), the 4 rays of a march CTA (4093) and the initial batch (4096), and
reach 65 537 with max_samples = 2^22, where truncation falls inside the batch.  Bitfields go through ngp_grid_update_bitfield so the
outer cascades are max-pooled as in training.  Coverage is asserted, not assumed: rays with more than MARCH_EMIT_CAP = 64 emitting
chunks (the re-march fallback of march_emit_kernel, read from the workspace), truncation, const_dt samples below 2^-10 and in the
binade [2^-10, 2^-9) where h / ulp is a tie, and emitting chunks that cross a power of two.  Compaction is checked with caps on both
sides of the live row count, so the zero-filled tail is compared too."""
import os

import numpy as np
import pytest
import torch

import march_ref as M
import oracle_lib as ol

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONE, NEAR, CASCADES = 0.00390625, 0.2, 5
LEGO = dict(aabb=(0.0, 1.0), const_dt=True)
FOX = dict(aabb=(-1.5, 2.5), const_dt=False)
EMIT_CAP = 64


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def npy(t):
    return t.detach().cpu().numpy()


def _raygen(ops, xf, focal, principal, W, H, n, seed):
    """n rays of random pixels of the cameras xf (n_img, 3, 4; NGP convention), through ops.raygen."""
    n_img = xf.shape[0]
    pix = np.random.default_rng(seed).integers(0, n_img * W * H, n).astype(np.int32)
    xf12 = np.ascontiguousarray(np.asarray(xf, np.float32).transpose(0, 2, 1)).reshape(n_img, 12)
    _, o, d = ops.raygen(cu(pix), W, H, cu(xf12), cu(np.tile(np.float32(focal), (n_img, 1))), cu(np.tile(np.float32(principal), (n_img, 1))))
    return npy(o), npy(d)


@pytest.fixture(scope="module")
def rays(ops):
    from jnerf_b200.plugin.dataset import NERF_SCALE, fov_to_focal_length, matrix_nerf2ngp, synthetic_cameras
    n = 65537
    W = H = 800
    f = fov_to_focal_length(W, 0.6911112070083618 * 180 / np.pi)
    xf = np.stack([matrix_nerf2ngp(m, NERF_SCALE, [0.5] * 3) for m in synthetic_cameras(100, seed=0)])
    lego = _raygen(ops, xf, (f, f), (0.5, 0.5), W, H, n, 1)
    c = np.load(os.path.join(ROOT, "tests", "golden", "fox_small", "capture.npz"))
    fl_x, fl_y, cx, cy, Wf, Hf = c["intrinsics"]
    mats = c["train_matrices"][c["train_present"]]
    assert int(c["aabb_scale"]) == 4
    xf = np.stack([matrix_nerf2ngp(m, NERF_SCALE, [0.5] * 3) for m in mats])
    fox = _raygen(ops, xf, (fl_x, fl_y), (cx / Wf, cy / Hf), int(Wf), int(Hf), n, 2)
    rng = np.random.default_rng(3)                                     # near = 0: origins inside the unit box, all directions
    o_in = rng.uniform(0.02, 0.98, (n, 3)).astype(np.float32)
    d_in = rng.normal(size=(n, 3))
    d_in = (d_in / np.linalg.norm(d_in, axis=1, keepdims=True)).astype(np.float32)
    return {"lego": lego, "fox": fox, "inside": (o_in, d_in)}


def _bitfield(ops, grid):
    g = cu(grid.astype(np.float32))
    mean = torch.zeros(1, dtype=torch.float32, device="cuda")
    bits = torch.zeros(M.G3 * CASCADES // 8, dtype=torch.uint8, device="cuda")
    ops.grid_update_bitfield(g, mean, bits, CASCADES)
    return npy(bits)


def _grid(kind, seed=0):
    rng = np.random.default_rng(seed)
    n = M.G3 * CASCADES
    if kind == "step0":                # a step-0 grid: every seen cell holds a small positive density, the mean is below every one of them
        return np.where(rng.random(n) < 0.98, np.float32(0.002), np.float32(0)).astype(np.float32)
    if kind == "shell":
        return ol.sphere_bitfield(0.3, shell=0.03)[1]
    if kind == "empty":
        return np.zeros(n, np.float32)
    if kind.startswith("speckle"):     # per-cascade random occupancy at density p
        p = float(kind[len("speckle"):])
        return (rng.random(n) < p).astype(np.float32)
    raise ValueError(kind)


@pytest.fixture(scope="module")
def bitfields(ops):
    cache = {}

    def get(kind):
        if kind not in cache:
            cache[kind] = _bitfield(ops, _grid(kind))
        return cache[kind]
    return get


def _gpu_march(ops, o, d, bits, cfg, max_samples, rng, near=NEAR, coords=None, ws=None):
    R = o.shape[0]
    if ws is None:
        ws = torch.empty(int(ops.lib.load().ngp_march_workspace_bytes(R)), dtype=torch.uint8, device="cuda")
    out = ops.march(cu(o), cu(d), cu(bits), cfg["aabb"], max_samples, CONE, near, CASCADES, cfg["const_dt"], rng, coords=coords, workspace=ws)
    torch.cuda.synchronize()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0                 # no producer / consumer hand-over timed out, error flag clear
    return out, ws


def _compare(gpu, ref):
    coords, ridx, numsteps, cnt = gpu
    rc, rr, rn, rk = ref
    assert np.array_equal(npy(cnt).view(np.uint32), rk)
    ns = npy(numsteps).view(np.uint32)
    assert np.array_equal(ns, rn)                                       # counts and ray-ordered bases
    assert np.array_equal(npy(ridx).view(np.uint32), rr)
    S = int(rn[:, 0].sum())                                             # rows of the accepted rays: a prefix of the buffer
    assert np.array_equal(npy(coords[:S]).view(np.uint32), rc[:S].view(np.uint32))
    return S


def _march_both(ops, o, d, bits, cfg, max_samples, near=NEAR, rng=None):
    rng = ol.pcg32_seed() if rng is None else rng
    gpu, ws = _gpu_march(ops, o, d, bits, cfg, max_samples, rng, near)
    ref = ol.march(o, d, bits, aabb=cfg["aabb"], max_samples=max_samples, cone_angle=CONE, near=near, cascades=CASCADES,
                   const_dt=cfg["const_dt"], rng=rng)
    S = _compare(gpu, ref)
    return gpu, ref, ws, S


@pytest.mark.parametrize("kind", ["step0", "shell", "speckle0.05", "speckle0.4", "empty"])
@pytest.mark.parametrize("scene", ["lego", "fox"])
@pytest.mark.parametrize("R", [1, 3, 1023, 1024, 1025, 4093, 4096])
def test_march_bit_exact_at_batch_sizes(ops, rays, bitfields, scene, kind, R):
    o, d = (a[:R] for a in rays[scene])
    _, ref, _, S = _march_both(ops, o, d, bitfields(kind), LEGO if scene == "lego" else FOX, R * 1024)
    if kind == "empty":
        assert S == 0 and (ref[1] == 0xFFFFFFFF).all()
    elif kind == "step0" and scene == "lego" and R >= 1023:
        assert (ref[2][:, 0] == 1024).any()                             # rays reach the 1024-step cap


@pytest.mark.parametrize("scene,kind", [("lego", "step0"), ("lego", "shell"), ("fox", "speckle0.05"), ("inside", "step0")])
def test_march_65537_rays_truncated(ops, rays, bitfields, scene, kind):
    o, d = rays[scene]
    R = o.shape[0]
    cfg = FOX if scene == "fox" else LEGO
    near = 0.0 if scene == "inside" else NEAR
    gpu, ref, _, S = _march_both(ops, o, d, bitfields(kind), cfg, 1 << 22, near=near)
    accepted = int(ref[3][0])
    print(f"[march] {scene}/{kind}: {accepted} / {R} rays accepted, {S} rows, {int(ref[3][1])} steps counted")
    if kind == "step0":
        assert 0 < accepted < R and int(ref[3][1]) > 1 << 22           # truncation falls inside the batch


def test_fallback_path_rays_over_64_emitting_chunks(ops, bitfields):
    """const_dt in the aabb_scale-16 box with speckled fine cascades: rays through the centre collect up to 1024 samples in short runs,
    spread over more than 64 chunks of 32 steps -- march_emit_kernel re-marches those rays with march_ray_warp<true>."""
    rng = np.random.default_rng(7)
    grid = np.zeros(M.G3 * CASCADES, np.float32)
    grid[:2 * M.G3] = (rng.random(2 * M.G3) < 0.25).astype(np.float32)   # cascades 0 and 1 speckled, the outer ones empty
    bits = _bitfield(ops, grid)
    R = 4096
    v = rng.normal(size=(R, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    o = (0.5 + 6.0 * v).astype(np.float32)
    t = 0.5 + rng.uniform(-0.3, 0.3, (R, 3)) - o
    d = (t / np.linalg.norm(t, axis=1, keepdims=True)).astype(np.float32)
    cfg = dict(aabb=(-7.5, 8.5), const_dt=True)
    gpu, ref, ws, S = _march_both(ops, o, d, bits, cfg, R * 1024)
    ne = M.n_emit(npy(ws), R)
    ns = ref[2]
    over = ne > EMIT_CAP
    print(f"[march] fallback: {int(over.sum())} of {R} rays with n_emit > {EMIT_CAP} (max {int(ne.max())}), {S} rows")
    assert over.sum() >= 10
    assert (ns[over, 0] > 0).all()
    rows_gpu = npy(gpu[0][:S]).view(np.uint32)
    for i in np.flatnonzero(over):                                      # those rays' rows, bit for bit (already part of _compare)
        b, n = int(ns[i, 1]), int(ns[i, 0])
        assert np.array_equal(rows_gpu[b:b + n], ref[0][b:b + n].view(np.uint32))


def test_const_dt_t_ranges_covered(ops, rays, bitfields):
    """near = 0 and origins inside the unit box: samples with t below 2^-10 and in the tie binade [2^-10, 2^-9), and emitting chunks whose
    32 steps cross a power of two (the closed form declines them, the sequential additions run) -- all bit-exact.  Each row is placed on
    its step of the ray's t sequence: tmin = 0 inside the box, so t_0 = fl(h * r) with the ray's jitter r, and t_k follows by float
    additions of h."""
    R = 4096
    o, d = (a[:R] for a in rays["inside"])
    _, ref, _, S = _march_both(ops, o, d, bitfields("step0"), LEGO, R * 1024, near=0.0)
    ns = ref[2]
    ray_of_row = np.repeat(np.arange(R), ns[:, 0])
    t = M.row_t(ref[0][:S], o[ray_of_row], d[ray_of_row], LEGO["aabb"])
    below, tie = int((t < 2.0 ** -10 * 0.999).sum()), int(((t > 2.0 ** -10 * 1.001) & (t < 2.0 ** -9 * 0.999)).sum())
    jitter = np.empty(R, np.float32)
    for i in range(R):                                                  # ray_setup: rng advanced by 8 per ray, one draw
        si = ol.pcg32_advance(ol.pcg32_seed(), i * 8)
        jitter[i] = ol.oracle().orc_pcg32_next_float(ol._ptr(si))
    t0 = (M.H_CONST.astype(np.float64) * jitter).astype(np.float32)     # fma(calc_dt(0), r, 0): one rounding of an exact product
    seq = M.sequential(t0, n=2048 + 64)                                 # the unit box's diagonal is 2048 steps
    k, err = M.step_of_rows(t, ray_of_row, seq)
    assert err < M.H_CONST / 16                                          # every row sits on one step of its ray's sequence
    emitting = np.zeros((R, seq.shape[1] // 32), bool)
    emitting[ray_of_row, k // 32] = True
    crossing = int((emitting & M.chunk_crosses_binade(seq)).sum())
    print(f"[march] const_dt: {below} samples with t < 2^-10, {tie} in [2^-10, 2^-9), {crossing} emitting chunks across a power of two "
          f"({int(emitting.sum())} emitting chunks)")
    assert below > 0 and tie > 0 and crossing > 1000


def test_workspace_reuse_smaller_batch(ops, rays, bitfields):
    """A smaller batch in the workspace and coords buffer of a larger one (DensityGridSampler._ensure_march_ws) equals a fresh march."""
    o, d = rays["lego"]
    bits = bitfields("step0")
    rng = ol.pcg32_seed()
    big, ws = _gpu_march(ops, o[:4096], d[:4096], bits, LEGO, 4096 * 1024, rng)
    coords = big[0]
    small, _ = _gpu_march(ops, o[4096:5121], d[4096:5121], bits, LEGO, 1025 * 1024, rng, coords=coords, ws=ws)
    fresh, _ = _gpu_march(ops, o[4096:5121], d[4096:5121], bits, LEGO, 1025 * 1024, rng)
    for a, b in zip(small[1:], fresh[1:]):
        assert torch.equal(a, b)
    S = int(npy(fresh[2])[:, 0].sum())
    assert torch.equal(small[0][:S], fresh[0][:S])
    _compare(fresh, ol.march(o[4096:5121], d[4096:5121], bits, max_samples=1025 * 1024, rng=rng))


@pytest.mark.parametrize("scene", ["lego", "fox"])
def test_data_parallel_shards(ops, rays, bitfields, scene):
    """rays[a:b] marched with the rng advanced by a * 8 (DensityGridSampler.sample_front): each ray's rows are the full batch's rows."""
    o, d = (x[:4096] for x in rays[scene])
    cfg = LEGO if scene == "lego" else FOX
    bits = bitfields("shell")
    full = ol.march(o, d, bits, aabb=cfg["aabb"], max_samples=4096 * 1024, cone_angle=CONE, near=NEAR, cascades=CASCADES, const_dt=cfg["const_dt"])
    fns = full[2]
    for a, b in ((0, 1500), (1500, 4093), (4093, 4096)):
        rng = ol.pcg32_advance(ol.pcg32_seed(), a * 8)
        gpu, _, _, _ = _march_both(ops, o[a:b], d[a:b], bits, cfg, (b - a) * 1024, rng=rng)   # counts, bases vs the shard's oracle march
        ns = npy(gpu[2]).view(np.uint32)
        assert np.array_equal(ns[:, 0], fns[a:b, 0])
        rows = npy(gpu[0]).view(np.uint32)
        for k in range(b - a):
            n = int(ns[k, 0])
            assert np.array_equal(rows[ns[k, 1]:ns[k, 1] + n], full[0][fns[a + k, 1]:fns[a + k, 1] + n].view(np.uint32))


def test_compaction_at_scale(ops, rays, bitfields):
    o, d = rays["lego"]
    gpu, ref, _, S = _march_both(ops, o, d, bitfields("shell"), LEGO, 1 << 22)
    ns = ref[2]
    long_rays = np.flatnonzero(ns[:, 0] > 5)
    mid = int(ns[long_rays[len(long_rays) // 2], 1]) + 3                  # a cap that falls inside a ray
    caps = [S + 5000, S, S - 1, mid, 1 << 18, 0]                          # S + 5000: a tail of 5000 rows past the live ones
    assert S > 1 << 18
    for cap in caps:
        rc, rn, rk = ol.compact(ref[0], ns, cap)                          # zero-initialised: its tail is the zero fill
        live = min(int(rk[0]), cap)
        assert (live < cap) == (cap > S)
        for alias in (False, True):
            if alias and cap > gpu[0].shape[0]:
                continue                                                  # an aliased compaction never asks for more rows than it has
            coords = gpu[0].clone()
            if not alias:                                                 # hand the output allocation a block full of NaN, not zeros
                junk = torch.full((cap, 7), float("nan"), device="cuda")
                del junk
            out, cns, ccnt = ops.compact(coords, gpu[2], cap, alias=alias)
            torch.cuda.synchronize()
            assert np.array_equal(npy(cns).view(np.uint32), rn) and np.array_equal(npy(ccnt).view(np.uint32), rk)
            if alias:
                assert out.data_ptr() == coords.data_ptr() and torch.equal(coords, gpu[0])    # bookkeeping only, rows untouched
                assert np.array_equal(npy(coords[:live]).view(np.uint32), rc[:live].view(np.uint32))
            else:
                assert out.shape == (cap, 7)                                                # live rows and the zero tail, bit for bit
                assert np.array_equal(npy(out).view(np.uint32), rc.view(np.uint32))
