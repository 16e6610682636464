"""Parity tests proper: every C-ABI operator of libngp_b200.so (sm_90a) against the oracle on identical seeded
inputs, and against the committed golden vectors.  Integer / index outputs (march, compaction, bitfields, sample
indices) must be bit-exact; floating point is checked at the tolerance stated beside each assert
(north_star: fp16/fp32 radiance within 1e-3 relative)."""
import os
import sys
import numpy as np
import pytest
import torch

import oracle_lib as ol

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_golden import digest, inputs, table  # noqa: E402

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "ngp_golden.npz"))
INP = inputs()


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


class device_scales:
    """Install the GPU-computed per-level scales into the oracle for the duration of a comparison (see
    orc_set_level_scales: the reference evaluates exp2f on the device)."""

    def __init__(self, lv):
        self.scales = np.ascontiguousarray(lv.table.cpu().numpy().view(np.float32).reshape(16, 8)[:, 0])

    def __enter__(self):
        ol.oracle().orc_set_level_scales(ol._ptr(self.scales))

    def __exit__(self, *a):
        ol.oracle().orc_set_level_scales(None)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def npy(t):
    return t.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------ R1
@pytest.mark.parametrize("aabb,log2T", [(1, 14), (1, 19), (4, 19)])
def test_level_table(ops, aabb, log2T):
    lv = ops.HashLevels(aabb, log2_hashmap_size=log2T)
    cfg = ol.HashCfg(aabb, log2_hashmap_size=log2T)
    assert np.array_equal(lv.offsets, cfg.offsets)
    tab = npy(lv.table).view(np.uint32).reshape(16, 8)
    scale = tab[:, 0].view(np.float32)
    for l in range(16):
        s_host = np.float32(np.exp2(np.float32(l) * cfg.log2_pls)) * np.float32(16) - np.float32(1)
        assert abs(scale[l] - s_host) <= 4 * np.spacing(np.float32(s_host))          # device exp2f: <= 2 ulp
        assert tab[l, 1] == int(np.ceil(s_host)) + 1                                   # resolution
        assert tab[l, 2] == cfg.offsets[l] and tab[l, 3] == cfg.offsets[l + 1] - cfg.offsets[l]
        dense = int(tab[l, 1]) ** 3 <= int(tab[l, 3])
        assert tab[l, 4] == (0 if dense else 1)


# ------------------------------------------------------------------------------------------------ R2 / R3
@pytest.mark.parametrize("log2T", [14, 19])
def test_hash_fwd_config1(ops, log2T):
    """BASELINE config #1: 4096 random points, L=16, T=2^14 (and the production T=2^19)."""
    lv = ops.HashLevels(1, log2_hashmap_size=log2T)
    cfg = ol.HashCfg(1, log2_hashmap_size=log2T)
    x = INP["x"].copy()
    x[0] = 0.0
    x[1] = 1.0
    for dt in (np.float32, np.float16):
        grid = table(cfg, dt)
        out = npy(ops.hash_fwd(cu(x), cu(grid), lv))
        with device_scales(lv):
            ref = ol.hash_fwd(cfg, x, grid, acc32=True) if dt == np.float16 else ol.hash_fwd(cfg, x, grid)
        # values are O(1e-4); fp32: reassociation-free fma chain -> 1e-9 abs; fp16: one rounding of an fp32 sum (<= 1 fp16 ulp)
        tol = 1e-9 if dt == np.float32 else 2.0 ** -11 * 2e-4
        assert np.abs(out.astype(np.float64) - ref.astype(np.float64)).max() <= tol
        if dt == np.float16:   # vs the reference's own fp16-accumulating arithmetic (golden, T=2^14): few fp16 ulps of 1e-4
            with device_scales(lv):
                ref16 = ol.hash_fwd(cfg, x, grid)
            assert np.abs(out.astype(np.float64) - ref16.astype(np.float64)).max() <= 8 * 2.0 ** -11 * 2e-4
    if log2T == 14:
        grid = table(cfg, np.float32)
        out = npy(ops.hash_fwd(cu(INP["x"]), cu(grid), lv))
        # golden from the reference's own source run on the host: libm exp2f scales (<= 2 ulp from the device's),
        # amplified by the finest resolution -> 2048 * 2^-23 * |table| ~ 5e-8
        assert np.abs(out[:256] - G["hash_fwd_f32_head"]).max() <= 1e-7


def test_hash_func_from_config(ops):
    """cfg.hash_func (HE/hash_encoder.py:13-16): another member of the XOR-of-products family, parsed into the level table's three
    multipliers -- forward and backward against the oracle evaluating the same expression."""
    from jnerf_b200.plugin.encoders import parse_hash_func
    primes = parse_hash_func("p1 * 2654435761 ^ p0 * 3 ^ 805459861 * p2")
    assert primes == (3, 2654435761, 805459861)
    cfg = ol.HashCfg(1, log2_hashmap_size=14)
    lv = ops.HashLevels(1, log2_hashmap_size=14, primes=primes)
    x = INP["x"]
    grid = table(cfg, np.float16)
    dy = INP["dy"].astype(np.float16)
    ol.oracle().orc_set_hash_primes(*primes)
    try:
        with device_scales(lv):
            ref = ol.hash_fwd(cfg, x, grid, acc32=True)
            gref = ol.hash_bwd(cfg, x, dy, acc32=True).astype(np.float64)
    finally:
        ol.oracle().orc_set_hash_primes(1, 19349663, 83492791)
    out = npy(ops.hash_fwd(cu(x), cu(grid), lv))
    assert np.abs(out.astype(np.float64) - ref.astype(np.float64)).max() <= 2.0 ** -11 * 2e-4
    default = npy(ops.hash_fwd(cu(x), cu(grid), ops.HashLevels(1, log2_hashmap_size=14)))
    assert np.abs(out.astype(np.float32) - default.astype(np.float32)).max() > 0          # the hashed levels really changed
    g = npy(ops.hash_bwd(cu(x), cu(dy), lv)).astype(np.float64)
    assert np.abs(g - gref).max() <= 2e-2 * np.abs(gref).max()


def test_hash_bwd(ops):
    cfg = ol.HashCfg(1, log2_hashmap_size=14)
    lv = ops.HashLevels(1, log2_hashmap_size=14)
    x = INP["x"]
    for dt in (np.float32, np.float16):
        dy = INP["dy"].astype(dt)
        g = npy(ops.hash_bwd(cu(x), cu(dy), lv)).astype(np.float64)
        with device_scales(lv):
            ref = ol.hash_bwd(cfg, x, dy, acc32=True).astype(np.float64) if dt == np.float16 else ol.hash_bwd(cfg, x, dy).astype(np.float64)
        scale = np.abs(ref).max()
        # fp32: atomic order only (1e-6 rel); fp16: each of up to ~100s of addends rounded to fp16 -> 2e-2 of the max
        tol = 1e-5 * scale if dt == np.float32 else 2e-2 * scale
        assert np.abs(g - ref).max() <= tol
        assert np.abs(g - ref).mean() <= tol * 0.05


# ------------------------------------------------------------------------------------------------ R4
def test_sh(ops):
    d = INP["dirs"]
    out = npy(ops.sh_fwd(cu(d), torch.float32))
    assert np.abs(out - ol.sh(d, np.float32)).max() <= 2e-6
    assert np.abs(out[:128] - G["sh_f32"]).max() <= 2e-6
    out16 = npy(ops.sh_fwd(cu(d), torch.float16)).astype(np.float32)
    assert np.abs(out16 - ol.sh(d, np.float16).astype(np.float32)).max() <= 2e-3


# ------------------------------------------------------------------------------------------------ R7
def _mlp_weights(nhm, seed):
    rng = np.random.default_rng(seed)
    shapes = [(64, 32)] + [(64, 64)] * nhm + [(16, 64)]
    lim = lambda s: np.sqrt(6.0 / (s[0] + s[1]))
    return np.concatenate([rng.uniform(-lim(s), lim(s), s).astype(np.float16).ravel() for s in shapes])


@pytest.mark.parametrize("nhm,n", [(0, 128), (1, 1000), (1, 65536), (2, 300)])
def test_mlp_fwd_bwd(ops, nhm, n):
    rng = np.random.default_rng(11)
    W = _mlp_weights(nhm, 2)
    X = np.clip(rng.standard_normal((n, 32)), -4, 4).astype(np.float16)
    Y, inter = ops.mlp_fwd(cu(W), cu(X), nhm)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    Yr, interr = ol.mlp_fwd(W, X, nhm)
    # fp32 accumulation in a different order + fp16 rounding of O(1) activations: 1 fp16 ulp (~1e-3 rel)
    assert np.abs(npy(inter).astype(np.float32) - interr.astype(np.float32)).max() <= 4e-3
    assert np.abs(npy(Y).astype(np.float32) - Yr.astype(np.float32)).max() <= 6e-3
    n_valid = 16 if nhm == 0 else 3
    dY = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    dY[:, n_valid:] = 0
    dX, temps, dW = ops.mlp_bwd(cu(W), cu(X), cu(interr), cu(dY), nhm, n_valid, need_dx=True, need_temps=True)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    dXr, tempsr, dWr = ol.mlp_bwd(W, X, interr, dY, nhm, n_valid)
    assert np.abs(npy(temps).astype(np.float32) - tempsr.astype(np.float32)).max() <= 3e-3
    assert np.abs(npy(dX).astype(np.float32) - dXr.astype(np.float32)).max() <= 3e-3
    dWg = npy(dW)
    assert np.abs(dWg - dWr).max() <= 2e-3 * max(1.0, np.abs(dWr).max())      # fp32 register accumulation vs float64
    off = 64 * 32 + nhm * 64 * 64
    assert (dWg[off + n_valid * 64:] == 0).all()


# ------------------------------------------------------------------------------------------------ fused network
def _net_inputs(n, seed=21, log2T=19, aabb=1):
    cfg = ol.HashCfg(aabb, log2_hashmap_size=log2T)
    rng = np.random.default_rng(seed)
    coords = np.zeros((n, 7), np.float32)
    coords[:, :3] = rng.random((n, 3), dtype=np.float32)
    coords[:, 3] = -0.0333333
    coords[:, 4:] = rng.random((n, 3), dtype=np.float32)
    grid = rng.uniform(-1, 1, cfg.n_params).astype(np.float16)               # O(1) features so the nets are exercised
    return cfg, coords, grid, _mlp_weights(0, 3), _mlp_weights(1, 4)


@pytest.mark.parametrize("n", [128, 1000, 40000])
def test_network_fwd(ops, n):
    cfg, coords, grid, Wd, Wr = _net_inputs(n)
    lv = ops.HashLevels(1)
    out, enc = ops.network_fwd(cu(coords), cu(grid), lv, cu(Wd), cu(Wr))
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    with device_scales(lv):
        ref, encr, hr = ol.network_fwd(cfg, coords[:, :3].copy(), coords[:, 4:].copy(), grid, Wd, Wr, acc32=True)
    assert np.abs(npy(enc).astype(np.float32) - encr.astype(np.float32)).max() <= 2e-3        # 1 fp16 ulp of O(1)
    d = np.abs(npy(out).astype(np.float32) - ref.astype(np.float32))
    assert d.max() <= 2e-2 and d.mean() <= 1e-3          # rare 1-ulp flips in hidden fp16 activations propagate
    sig = npy(ops.density_fwd(cu(coords[:, :3].copy()), cu(grid), lv, cu(Wd))).astype(np.float32)
    assert np.abs(sig - hr[:, 0].astype(np.float32)).max() <= 1e-2


def test_network_fwd_live_count(ops):
    cfg, coords, grid, Wd, Wr = _net_inputs(1000)
    lv = ops.HashLevels(1)
    out = torch.full((1000, 4), 7.0, dtype=torch.float16, device="cuda")
    n_dev = torch.tensor([300], dtype=torch.int32, device="cuda")
    ops.network_fwd(cu(coords), cu(grid), lv, cu(Wd), cu(Wr), n_dev=n_dev, out=out)
    full, _ = ops.network_fwd(cu(coords), cu(grid), lv, cu(Wd), cu(Wr))
    assert torch.equal(out[:300], full[:300]) and (out[300:] == 7.0).all()      # rows past the live count, in its tile too, untouched


@pytest.mark.parametrize("aabb,log2T", [(1, 14), (1, 19), (4, 19)])
def test_network_bwd(ops, aabb, log2T):
    """(1,14): BASELINE config #1's table; (1,19): the production lego table; (4,19): the fox table (ngp_fox.py, aabb_scale 4)."""
    n = 3000
    cfg, coords, grid, Wd, Wr = _net_inputs(n, log2T=log2T, aabb=aabb)
    lv = ops.HashLevels(aabb, log2_hashmap_size=log2T)
    rng = np.random.default_rng(5)
    dout = (rng.standard_normal((n, 4)) * 0.05).astype(np.float16)
    out, enc = ops.network_fwd(cu(coords), cu(grid), lv, cu(Wd), cu(Wr))
    gg = torch.zeros(cfg.n_params, dtype=torch.float16, device="cuda")
    dwd = torch.zeros(Wd.size, dtype=torch.float32, device="cuda")
    dwr = torch.zeros(Wr.size, dtype=torch.float32, device="cuda")
    ops.network_bwd(cu(coords), enc, lv, cu(Wd), cu(Wr), cu(dout), gg, dwd, dwr)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    # oracle chain: same math layer by layer
    pos, dirs = coords[:, :3].copy(), coords[:, 4:].copy()
    _, encr, h = ol.network_fwd(cfg, pos, dirs, grid, Wd, Wr, acc32=True)
    encr = npy(enc)                                             # start both chains from the same fp16 features
    h, inter_d = ol.mlp_fwd(Wd, encr, 0)
    rin = np.concatenate([h, ol.sh(dirs, np.float16)], 1)
    r, inter_r = ol.mlp_fwd(Wr, rin, 1)
    dYr = np.zeros((n, 16), np.float16)
    dYr[:, :3] = dout[:, :3]
    d_rin, _, dWr_ref = ol.mlp_bwd(Wr, rin, inter_r, dYr, 1, 3)
    dYd = d_rin[:, :16].astype(np.float32)
    dYd[:, 0] += dout[:, 3].astype(np.float32)
    dYd = dYd.astype(np.float16)
    d_enc, _, dWd_ref = ol.mlp_bwd(Wd, encr, inter_d, dYd, 0, 16)
    with device_scales(lv):
        gg_ref = ol.hash_bwd(cfg, pos, d_enc, acc32=True)
    sW = max(np.abs(dWr_ref).max(), np.abs(dWd_ref).max())
    assert np.abs(npy(dwr) - dWr_ref).max() <= 2e-2 * sW and np.abs(npy(dwd) - dWd_ref).max() <= 2e-2 * sW
    g = npy(gg).astype(np.float64)
    sG = np.abs(gg_ref).max()
    assert np.abs(g - gg_ref).max() <= 5e-2 * sG and np.abs(g - gg_ref).mean() <= 2e-3 * sG


# ------------------------------------------------------------------------------------------------ R5 / R6
@pytest.mark.parametrize("const_dt", [True, False])
def test_march_bit_exact(ops, const_dt):
    bits, _ = ol.sphere_bitfield(0.3)
    aabb = (0.0, 1.0) if const_dt else (-1.5, 2.5)
    tag = "constdt" if const_dt else "cone"
    o, d = INP["rays_o"], INP["rays_d"]
    rng = ol.pcg32_seed()
    coords, ridx, numsteps, cnt = ops.march(cu(o), cu(d), cu(bits), aabb, 300 * 1024, 0.00390625, 0.2, 5, const_dt, rng)
    ref = ol.march(o, d, bits, aabb=aabb, const_dt=const_dt, max_samples=300 * 1024)     # GPU arithmetic (fma_mode 1)
    S = int(ref[3][1])
    assert np.array_equal(npy(cnt).view(np.uint32), ref[3])
    assert np.array_equal(npy(numsteps).view(np.uint32), ref[2])                          # counts and ray-ordered bases
    assert np.array_equal(npy(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32))    # every sample, bit for bit
    assert np.array_equal(npy(ridx).view(np.uint32), ref[1])
    # golden (host arithmetic of the reference source): identical step counts for all but FMA-boundary rays
    gold = G[f"march_{tag}_numsteps"]
    assert (npy(numsteps).view(np.uint32)[:, 0] != gold[:, 0]).mean() <= 0.02


def test_march_overflow_and_compact(ops):
    bits, _ = ol.sphere_bitfield(0.3)
    o, d = INP["rays_o"], INP["rays_d"]
    rng = ol.pcg32_seed()
    a = ops.march(cu(o), cu(d), cu(bits), (0.0, 1.0), 2000, 0.00390625, 0.2, 5, True, rng)
    b = ol.march(o, d, bits, max_samples=2000)
    assert np.array_equal(npy(a[2]).view(np.uint32), b[2]) and np.array_equal(npy(a[3]).view(np.uint32), b[3])
    full = ops.march(cu(o), cu(d), cu(bits), (0.0, 1.0), 300 * 1024, 0.00390625, 0.2, 5, True, rng)
    ref = ol.march(o, d, bits, max_samples=300 * 1024)
    S = int(ref[3][1])
    cc, ns, cnt = ops.compact(full[0], full[2], S - 777)
    rc = ol.compact(ref[0], ref[2], S - 777)
    assert np.array_equal(npy(ns).view(np.uint32), rc[1]) and np.array_equal(npy(cnt).view(np.uint32), rc[2])
    assert np.array_equal(npy(cc).view(np.uint32), rc[0].view(np.uint32))
    _, ns2, cnt2 = ops.compact(full[0], full[2], S - 777, alias=True)
    assert torch.equal(ns2, ns) and torch.equal(cnt2, cnt)


# ------------------------------------------------------------------------------------------------ R8 / R9
@pytest.mark.parametrize("dt", [np.float32, np.float16])
def test_composite(ops, dt):
    bits, _ = ol.sphere_bitfield(0.3)
    o, d = INP["rays_o"], INP["rays_d"]
    coords, _, numsteps, cnt = ol.march(o, d, bits, max_samples=300 * 1024)
    S = int(cnt[1])
    cc, ns_c, _ = ol.compact(coords, numsteps, S - 777)
    rng = np.random.default_rng(8)
    net = rng.standard_normal((S - 777, 4)).astype(np.float32).astype(dt)
    bg = rng.random((300, 3), dtype=np.float32)
    lg = rng.standard_normal((300, 3)).astype(np.float32)
    numsteps_i, ns_ci = numsteps.view(np.int32), ns_c.view(np.int32)
    rgb = npy(ops.composite_fwd(cu(net), cu(cc), cu(numsteps_i), cu(ns_ci), cu(bg)))
    rgb_ref = ol.composite_fwd(net, cc, numsteps, ns_c, bg)
    assert np.abs(rgb - rgb_ref).max() <= 1e-3 * max(1.0, np.abs(rgb_ref).max())            # __expf vs expf
    tag = "f32" if dt == np.float32 else "f16"
    assert np.abs(rgb - G[f"comp_{tag}_rgb"]).max() <= 1e-3                                  # reference-source golden
    mean = torch.tensor([0.001], dtype=torch.float32, device="cuda")
    dnet = npy(ops.composite_bwd(cu(net), cu(cc), cu(ns_ci), cu(lg), cu(rgb_ref), mean)).astype(np.float32)
    dref = ol.composite_bwd(net, cc, ns_c, lg, rgb_ref, 0.001).astype(np.float32)
    assert np.abs(dnet - dref).max() <= 2e-3 * np.abs(dref).max() + 1e-6
    assert np.abs(dnet[:64] - G[f"comp_{tag}_dnet_head"].astype(np.float32)).max() <= 2e-3 * np.abs(dref).max() + 1e-6
    rgbi, alpha = ops.composite_infer(cu(net), cu(cc), cu(ns_ci))
    ri, ai = ol.composite_infer(net, cc, ns_c)
    assert np.abs(npy(rgbi) - ri).max() <= 1e-3 and np.abs(npy(alpha) - ai).max() <= 1e-3
    if dt == np.float16:
        target = rng.random((300, 3), dtype=np.float32)
        rgb2, loss, dnet2 = ops.composite_loss_bwd(cu(net), cu(cc), cu(numsteps_i), cu(ns_ci), cu(bg), cu(target), mean)
        g, l = ol.huber_grad(rgb_ref, target)
        dref2 = ol.composite_bwd(net, cc, ns_c, g.reshape(300, 3), rgb_ref, 0.001).astype(np.float32)
        assert np.abs(npy(rgb2) - rgb_ref).max() <= 1e-3
        assert np.abs(npy(loss) - l.reshape(300, 3).sum(1)).max() <= 2e-3
        assert np.abs(npy(dnet2).astype(np.float32) - dref2).max() <= 3e-3 * np.abs(dref2).max() + 1e-6


# ------------------------------------------------------------------------------------------------ R10
def test_grid_maintenance(ops):
    rng = np.random.default_rng(9)
    n_el = ol.G3 * 5
    g_in = np.where(rng.random(n_el) < 0.3, rng.random(n_el) * 0.05, -1.0).astype(np.float32)
    si = ol.pcg32_seed()
    n = 20000
    step = torch.tensor([3], dtype=torch.int32, device="cuda")
    pos, idx = ops.grid_generate_samples(n, si, step, (-1.5, 2.5), cu(g_in), 3, 0.01)
    pr, ir = ol.generate_grid_samples(n, si, 3, (-1.5, 2.5), g_in, 3, 0.01)
    assert np.array_equal(npy(idx).view(np.uint32), ir)                                      # cell indices: bit-exact
    assert np.array_equal(digest(npy(idx).view(np.uint32)), G["gridgen_idx_sha"])            # and equal to the golden
    assert np.array_equal(npy(pos), pr)                                                      # positions: same float ops
    mlp = rng.standard_normal(n).astype(np.float32)
    tmp = torch.zeros(n_el, dtype=torch.float32, device="cuda")
    ops.grid_splat(idx, cu(mlp), tmp)
    tr = np.zeros(n_el, np.float32)
    ol.splat(ir, mlp, tr)
    assert np.abs(npy(tmp) - tr).max() <= 1e-6 * tr.max() + 1e-9                             # __expf vs expf
    grid = cu(g_in)
    ops.grid_ema(grid, cu(tr))
    gr = g_in.copy()
    ol.ema(gr, tr)
    assert np.array_equal(npy(grid), gr)
    mean = torch.zeros(1, dtype=torch.float32, device="cuda")
    bits = torch.zeros(n_el // 8, dtype=torch.uint8, device="cuda")
    ops.grid_update_bitfield(grid, mean, bits)
    m_ref = ol.grid_mean(gr)
    assert abs(float(mean.item()) - m_ref) <= 1e-5 * m_ref
    assert np.array_equal(npy(bits), ol.update_bitfield(gr, float(mean.item())))            # bitfield: bit-exact given the mean
    # mark_untrained
    n_img = 7
    xf = np.zeros((n_img, 12), np.float32)
    r2 = np.random.default_rng(9)
    for j in range(n_img):
        v = r2.normal(size=3); v /= np.linalg.norm(v)
        zc = -v
        xc = np.cross(np.array([0, 0, 1.0]), zc); xc /= np.linalg.norm(xc)
        xf[j] = np.concatenate([xc, np.cross(zc, xc), zc, 0.5 + 1.2 * v]).astype(np.float32)
    focal = np.full((n_img, 2), 1100.0, np.float32)
    ga = torch.zeros(n_el, dtype=torch.float32, device="cuda")
    ops.grid_mark_untrained(ga, cu(focal), cu(xf), (800, 800))
    gb = np.zeros(n_el, np.float32)
    ol.oracle().orc_set_fma_mode(0)
    ol.mark_untrained(gb, focal, xf, (800, 800))
    ol.oracle().orc_set_fma_mode(1)
    assert np.array_equal(npy(ga), gb)


# ------------------------------------------------------------------------------------------------ N1 / N2
def test_adam_ema(ops):
    rng = np.random.default_rng(5)
    n = 100003
    for pdt, gdt in ((np.float16, np.float16), (np.float16, np.float32), (np.float32, np.float32)):
        p0 = rng.uniform(-1e-1, 1e-1, n).astype(pdt)
        master = p0.astype(np.float32)
        p, m, v, ms = cu(p0), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), cu(master)
        pr, mr, vr, msr = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32), master.copy()
        for step in range(1, 5):
            g = (rng.standard_normal(n) * 1e-3).astype(gdt)
            gt = cu(g)
            ops.adam_ema(p, gt, m, v, ms, 0.1, step)
            assert (gt == 0).all()
            ol.adam_ema(pr, g.astype(np.float32), mr, vr, msr, 0.1, step)
            assert np.abs(npy(ms) - msr).max() <= 1e-5 and np.abs(npy(p).astype(np.float32) - pr.astype(np.float32)).max() <= 2.5e-4   # <= 1 fp16 ulp at |p| < 0.25


def test_raygen(ops):
    rng = np.random.default_rng(6)
    n_img, W, H = 5, 64, 48
    xf = rng.standard_normal((n_img, 12)).astype(np.float32)
    focal = np.full((n_img, 2), 70.0, np.float32)
    pp = np.full((n_img, 2), 0.5, np.float32)
    pix = rng.integers(0, n_img * W * H, 5000).astype(np.int32)
    img, o, d = ops.raygen(cu(pix), W, H, cu(xf), cu(focal), cu(pp))
    ir, orr, dr = ol.raygen(pix.view(np.uint32), W, H, xf, focal, pp)
    assert np.array_equal(npy(img).view(np.uint32), ir) and np.array_equal(npy(o), orr)
    assert np.abs(npy(d) - dr).max() <= 1e-6


def test_prepare_batch(ops):
    rng = np.random.default_rng(6)
    n_img, W, H = 3, 32, 24
    xf = rng.standard_normal((n_img, 12)).astype(np.float32)
    focal = np.full((n_img, 2), 40.0, np.float32)
    pp = np.full((n_img, 2), 0.5, np.float32)
    pix = rng.integers(0, n_img * W * H, 1000).astype(np.int32)
    bg = rng.random((1000, 3), dtype=np.float32)
    for dt in (np.uint8, np.float32):
        img = rng.integers(0, 256, (n_img * W * H, 4)).astype(np.uint8)
        imgf = img.astype(np.float32) / 255.0
        images = img if dt == np.uint8 else imgf
        ids, o, d, target = ops.prepare_batch(cu(pix), W, H, cu(xf), cu(focal), cu(pp), cu(images), cu(bg))
        ir, orr, dr = ol.raygen(pix.view(np.uint32), W, H, xf, focal, pp)
        c = imgf[pix]
        tref = c[:, :3] * c[:, 3:] + bg * (1 - c[:, 3:])                                   # runner/runner.py:68
        assert np.array_equal(npy(ids).view(np.uint32), ir) and np.array_equal(npy(o), orr) and np.abs(npy(d) - dr).max() <= 1e-6
        assert np.abs(npy(target) - tref).max() <= 1e-6


@pytest.mark.gpu
def test_dp_exchange_kernel_two_ranks_on_one_device(ops):
    """ngp_dp_exchange_step with two emulated ranks (two arenas, two streams, one GPU): the flag hand-shake completes, every
    rank ends with the same table == ngp_adam_ema applied to the summed gradients, for two consecutive epochs."""
    from jnerf_b200 import dp
    W, n, n_w = 2, 400_003, 10240
    arenas = [dp.PeerArena(n, n_w, W, r, None, ipc=False) for r in range(W)]
    for a in arenas:
        a.base = [b.buf.data_ptr() for b in arenas]
    P = arenas[0].P
    sl = P // W
    g = torch.Generator(device="cuda").manual_seed(5)
    table0 = torch.zeros(P, device="cuda")
    table0[:n] = torch.rand(n, device="cuda", generator=g) * 2e-4 - 1e-4
    w0 = (torch.randn(n_w, device="cuda", generator=g) * 0.1)
    state = []
    for r, a in enumerate(arenas):
        a.table.copy_(table0.half())
        state.append(dict(m=torch.zeros(sl, device="cuda"), v=torch.zeros(sl, device="cuda"), master=table0.half().float()[r * sl:(r + 1) * sl].clone(),
                          w=w0.half().clone(), wm=torch.zeros(n_w, device="cuda"), wv=torch.zeros(n_w, device="cuda"), wmaster=w0.half().float().clone()))
    # reference: one plain Adam+EMA over the whole table / weight vector with the summed gradient
    ref = dict(p=table0.half().clone(), m=torch.zeros(P, device="cuda"), v=torch.zeros(P, device="cuda"), master=table0.half().float().clone(),
               w=w0.half().clone(), wm=torch.zeros(n_w, device="cuda"), wv=torch.zeros(n_w, device="cuda"), wmaster=w0.half().float().clone())
    streams = [torch.cuda.Stream() for _ in range(W)]
    for epoch in (1, 2):
        gsum, wsum = torch.zeros(P, device="cuda"), torch.zeros(n_w, device="cuda")
        for a in arenas:
            a.table_grad[:n].copy_((torch.randn(n, device="cuda", generator=g) * 1e-3).half())
            a.w_grad[:n_w].copy_(torch.randn(n_w, device="cuda", generator=g) * 1e-2)
            gsum += a.table_grad.float()
            wsum += a.w_grad[:n_w]
        torch.cuda.synchronize()
        for r, a in enumerate(arenas):
            st = state[r]
            with torch.cuda.stream(streams[r]):
                ops.dp_exchange_step(W, r, sl, n_w, a.peers("table"), a.peers("table_grad"), a.peers("w_grad"), a.peers("flags"), epoch,
                                     st["m"], st["v"], st["master"], st["w"], st["wm"], st["wv"], st["wmaster"], 0.1, epoch, grad_scale=0.5)
                ops.dp_exchange_wait(W, a.flags, epoch)
                a.grads.zero_()
        torch.cuda.synchronize()
        ops.adam_ema(ref["p"], gsum, ref["m"], ref["v"], ref["master"], 0.1, epoch, grad_scale=0.5, zero_grad=False)
        ops.adam_ema(ref["w"], wsum, ref["wm"], ref["wv"], ref["wmaster"], 0.1, epoch, grad_scale=0.5, zero_grad=False)
        torch.cuda.synchronize()
        for r, a in enumerate(arenas):
            assert torch.equal(a.table, ref["p"]), f"epoch {epoch}: table of rank {r} differs"
            assert torch.equal(state[r]["w"], ref["w"]), f"epoch {epoch}: MLP weights of rank {r} differ"
            assert torch.equal(state[r]["master"], ref["master"][r * sl:(r + 1) * sl])
            assert int(a.table_grad.abs().sum()) == 0 and int(a.flags[32]) == 0
