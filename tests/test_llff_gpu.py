"""Six and seven occupancy cascades on the H100 (aabb_scale 32: LLFFDataset's default; 64: ngp_llff.py), the regime a forward-facing
LLFF capture trains in: every sampler / grid / composite operator against the oracle with the cascade count passed through, the
aabb_scale-64 hash table through the standalone and the fused network kernels, and runner.llff_cfg end to end on the forward-facing
stand-in (write_synthetic_llff -> LLFFDataset).  Integer outputs are bit-exact; floating point at the tolerances of test_gpu_ops.py
and test_gpu_parity_e2e.py."""
import os

import numpy as np
import pytest
import torch

import oracle_lib as ol
from test_gpu_ops import _mlp_weights, cu, device_scales, npy
from test_llff_cpu import G3, shells_bitfield, update_bitfield, wide_rays

pytestmark = pytest.mark.gpu

CASCADES = [6, 7]


def aabb_of(cascades):
    scale = 1 << (cascades - 1)
    return (0.5 - scale / 2, 0.5 + scale / 2)


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def scenes():
    """cascades -> (bitfield, density grid) with occupied cells in every cascade."""
    return {c: shells_bitfield(c) for c in CASCADES}


def oracle_march(o, d, bits, cascades, const_dt, cap, rng=None):
    return ol.march(o, d, bits, aabb=aabb_of(cascades), max_samples=cap, cascades=cascades, const_dt=const_dt, rng=rng)


# ------------------------------------------------------------------------------------------------ 7. ray generation
def test_raygen_on_an_llff_batch(ops, tmp_path):
    """ngp_raygen on a shuffled LLFFDataset batch against generate_random_data (llff_dataset.py:291-308) restated with numpy."""
    from jnerf_b200.plugin import dataset as D
    D.write_synthetic_llff(str(tmp_path), n_images=9, H=60, W=80, seed=3)
    ds = D.LLFFDataset(str(tmp_path), 2048, mode="train", factor=1, llffhold=4, aabb_scale=64, seed=5)
    pix = ds.next_pixels()
    ids, o, d, rgba = ds.rays_for(pix) + (ds.rgba_for(pix),)
    p = npy(pix).astype(np.int64)
    H, W = ds.H, ds.W
    img_id, off = p // (H * W), p % (H * W)
    xf = npy(ds.transforms_gpu)[img_id].reshape(-1, 4, 3).transpose(0, 2, 1).astype(np.float64)
    xy = np.stack([((off % W) + 0.5) / W, ((off // W) + 0.5) / H], -1)
    dc = np.concatenate([(xy - npy(ds.metadata)[img_id, 4:6]) * np.array([W, H]) / npy(ds.focal_lengths)[img_id], np.ones((len(p), 1))], -1)
    dw = np.einsum("nij,nj->ni", xf[:, :, :3], dc)
    dw /= np.linalg.norm(dw, axis=1, keepdims=True)
    assert np.array_equal(npy(ids).astype(np.int64), img_id) and np.array_equal(npy(o), xf[:, :, 3].astype(np.float32))
    assert np.abs(npy(d) - dw).max() <= 1e-6
    assert np.abs(npy(rgba) - npy(ds.image_data).reshape(-1, 4)[p].astype(np.float32) / 255).max() <= 1e-7     # the stored bytes / 255


# ------------------------------------------------------------------------------------------------ 8. march
@pytest.mark.parametrize("const_dt", [True, False])
@pytest.mark.parametrize("cascades", CASCADES)
def test_march_bit_exact(ops, scenes, cascades, const_dt):
    bits, _ = scenes[cascades]
    per = bits.reshape(cascades, -1)
    assert all(int(np.count_nonzero(per[k])) > 0 for k in range(cascades))
    R = 300
    o, d = wide_rays(R, cascades, seed=cascades)
    rng = ol.pcg32_seed()
    cap = R * 1024
    coords, ridx, numsteps, cnt = ops.march(cu(o), cu(d), cu(bits), aabb_of(cascades), cap, 0.00390625, 0.2, cascades, const_dt, rng)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    ref = oracle_march(o, d, bits, cascades, const_dt, cap)
    S = int(ref[3][1])
    assert np.array_equal(npy(cnt).view(np.uint32), ref[3])
    assert np.array_equal(npy(numsteps).view(np.uint32), ref[2])                          # counts and ray-ordered bases
    assert np.array_equal(npy(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32))    # every sample, bit for bit
    assert np.array_equal(npy(ridx).view(np.uint32), ref[1])
    ns = ref[2][:, 0]
    assert S > 10 * R and (ns[0::3] > 0).any() and (ns[2::3] > 0).any()                   # rays from inside and from far outside sample
    if not const_dt:
        # cone stepping reaches step sizes only the outer cascades allow: dt above the 5-cascade maximum occurs
        min_cone = np.sqrt(3.0) / 1024
        dt = ref[0][:S, 3] * (min_cone * (1 << (cascades - 1)) - min_cone) + min_cone     # nerf_unwarp_dt
        assert dt.max() > min_cone * 16 * 1.5


@pytest.mark.parametrize("const_dt", [True, False])
@pytest.mark.parametrize("cascades", CASCADES)
def test_whole_frame_renderer_sample_counts_equal_the_march(ops, scenes, cascades, const_dt):
    """test_render_gpu.py's check at 5 cascades: ngp_render_* under the jitter layout of the tiled march, min_transmittance 0."""
    bits, _ = scenes[cascades]
    R, tile = 1500, 512
    o, d = wide_rays(R, cascades, seed=10 + cascades)
    o, d, b = cu(o), cu(d), cu(bits)
    aabb_scale = 1 << (cascades - 1)
    lv = ops.HashLevels(aabb_scale)
    g = torch.Generator(device="cuda").manual_seed(2)
    grid = ((torch.rand(lv.n_params, device="cuda", generator=g) * 2 - 1) * 0.1).half()
    Wd, Wr = cu(_mlp_weights(0, 3)), cu(_mlp_weights(1, 4))
    rng = ol.pcg32_seed()
    rgb, alpha, n, rounds = ops.render_rays(o, d, b, aabb_of(cascades), 0.00390625, 0.2, cascades, const_dt, rng, grid, lv, Wd, Wr, tile,
                                            min_transmittance=0.0)
    st, want = rng.copy(), []
    for p in range(0, R, tile):
        _, _, numsteps, _ = ops.march(o[p:p + tile].contiguous(), d[p:p + tile].contiguous(), b, aabb_of(cascades), tile * 1024, 0.00390625, 0.2,
                                      cascades, const_dt, st)
        ops.pcg32_advance(st)
        want.append(numsteps[:, 0].cpu())
    want = torch.cat(want)
    assert torch.equal(n.cpu().to(want.dtype), want) and int(want.sum()) > 10 * R and rounds >= 1
    assert torch.isfinite(rgb).all() and torch.isfinite(alpha).all()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0


# ------------------------------------------------------------------------------------------------ 9. composite
@pytest.mark.parametrize("cascades", CASCADES)
def test_composite_with_dt_warped_at_these_cascades(ops, scenes, cascades):
    bits, _ = scenes[cascades]
    R = 300
    o, d = wide_rays(R, cascades, seed=20 + cascades)
    coords, _, numsteps, cnt = oracle_march(o, d, bits, cascades, False, R * 1024)            # cone stepping: dt varies along a ray
    S = int(cnt[1])
    cc, ns_c, _ = ol.compact(coords, numsteps, S - 555)
    rng = np.random.default_rng(8)
    bg = rng.random((R, 3), dtype=np.float32)
    lg = rng.standard_normal((R, 3)).astype(np.float32)
    numsteps_i, ns_ci = numsteps.view(np.int32), ns_c.view(np.int32)
    mean = torch.tensor([0.001], dtype=torch.float32, device="cuda")
    for dt in (np.float32, np.float16):
        net = rng.standard_normal((S - 555, 4)).astype(np.float32).astype(dt)
        rgb = npy(ops.composite_fwd(cu(net), cu(cc), cu(numsteps_i), cu(ns_ci), cu(bg), cascades))
        rgb_ref = ol.composite_fwd(net, cc, numsteps, ns_c, bg, cascades)
        assert np.abs(rgb - rgb_ref).max() <= 1e-3 * max(1.0, np.abs(rgb_ref).max())            # __expf vs expf
        # the cascade count matters: the same rows composited with the 5-cascade dt warp give another image
        assert np.abs(ol.composite_fwd(net, cc, numsteps, ns_c, bg, 5) - rgb_ref).max() > 1e-2
        dnet = npy(ops.composite_bwd(cu(net), cu(cc), cu(ns_ci), cu(lg), cu(rgb_ref), mean, cascades)).astype(np.float32)
        dref = ol.composite_bwd(net, cc, ns_c, lg, rgb_ref, 0.001, cascades).astype(np.float32)
        assert np.abs(dnet - dref).max() <= 2e-3 * np.abs(dref).max() + 1e-6
        rgbi, alpha = ops.composite_infer(cu(net), cu(cc), cu(ns_ci), cascades)
        ri, ai = ol.composite_infer(net, cc, ns_c, cascades)
        assert np.abs(npy(rgbi) - ri).max() <= 1e-3 and np.abs(npy(alpha) - ai).max() <= 1e-3
    target = rng.random((R, 3), dtype=np.float32)
    rgb2, loss, dnet2 = ops.composite_loss_bwd(cu(net), cu(cc), cu(numsteps_i), cu(ns_ci), cu(bg), cu(target), mean, cascades=cascades)
    g, l = ol.huber_grad(rgb_ref, target)
    dref2 = ol.composite_bwd(net, cc, ns_c, g.reshape(R, 3), rgb_ref, 0.001, cascades).astype(np.float32)
    assert np.abs(npy(rgb2) - rgb_ref).max() <= 1e-3
    assert np.abs(npy(loss) - l.reshape(R, 3).sum(1)).max() <= 2e-3
    assert np.abs(npy(dnet2).astype(np.float32) - dref2).max() <= 3e-3 * np.abs(dref2).max() + 1e-6


# ------------------------------------------------------------------------------------------------ 10. occupancy grid
@pytest.mark.parametrize("cascades", CASCADES)
def test_grid_update(ops, cascades):
    rng = np.random.default_rng(9)
    n_el = G3 * cascades
    aabb = aabb_of(cascades)
    # mark_untrained over all cascades: cameras of a forward-facing capture, close to the centre and looking one way
    n_img = 7
    xf = np.zeros((n_img, 12), np.float32)
    for j in range(n_img):
        zc = np.array([0.2 * rng.normal(), 0.2 * rng.normal(), 1.0])
        zc /= np.linalg.norm(zc)
        xc = np.cross(np.array([0, 1.0, 0]), zc)
        xc /= np.linalg.norm(xc)
        xf[j] = np.concatenate([xc, np.cross(zc, xc), zc, 0.5 + 0.15 * rng.normal(size=3)]).astype(np.float32)
    focal = np.full((n_img, 2), 408.0, np.float32)
    ga = torch.zeros(n_el, dtype=torch.float32, device="cuda")
    ops.grid_mark_untrained(ga, cu(focal), cu(xf), (504, 378))
    gb = np.zeros(n_el, np.float32)
    ol.oracle().orc_set_fma_mode(0)
    ol.mark_untrained(gb, focal, xf, (504, 378))
    ol.oracle().orc_set_fma_mode(1)
    assert np.array_equal(npy(ga), gb)
    per = gb.reshape(cascades, G3)
    assert all(0 < int((per[k] < 0).sum()) < G3 for k in range(cascades))                      # seen and unseen cells in every cascade
    # sample generation over max_cascade + 1 = `cascades` levels, on a grid with trained and untrained cells
    g_in = np.where(rng.random(n_el) < 0.3, rng.random(n_el) * 0.05, -1.0).astype(np.float32)
    si = ol.pcg32_seed()
    n = 60000
    step = torch.tensor([3], dtype=torch.int32, device="cuda")
    parts = []
    for thresh in (-0.01, 0.01):                                                                # uniform and occupied-only draws
        pos, idx = ops.grid_generate_samples(n, si, step, aabb, cu(g_in), cascades, thresh)
        pr, ir = ol.generate_grid_samples(n, si, 3, aabb, g_in, cascades, thresh)
        assert np.array_equal(npy(idx).view(np.uint32), ir) and np.array_equal(npy(pos), pr)
        assert sorted(set((ir // G3).tolist())) == list(range(cascades))                        # every level drawn, the outermost included
        assert pr.min() >= 0 and pr.max() <= 1 and np.abs(pr - 0.5).max() > 0.4                 # positions leave warped to the aabb's unit cube
        ol.pcg32_advance(si)
        parts.append((idx, ir))
    idx, ir = torch.cat([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    mlp = rng.standard_normal(2 * n).astype(np.float32)
    tmp = torch.zeros(n_el, dtype=torch.float32, device="cuda")
    ops.grid_splat(idx, cu(mlp), tmp)
    tr = np.zeros(n_el, np.float32)
    ol.splat(ir, mlp, tr)
    assert np.abs(npy(tmp) - tr).max() <= 1e-6 * tr.max() + 1e-9                                # __expf vs expf
    assert float(tr[(cascades - 1) * G3:].max()) > 0
    grid = cu(g_in)
    ops.grid_ema(grid, cu(tr))
    gr = g_in.copy()
    ol.ema(gr, tr)
    assert np.array_equal(npy(grid), gr)
    mean = torch.zeros(1, dtype=torch.float32, device="cuda")
    bits = torch.zeros(n_el // 8, dtype=torch.uint8, device="cuda")
    ops.grid_update_bitfield(grid, mean, bits, cascades)
    m_ref = ol.grid_mean(gr)
    assert abs(float(mean.item()) - m_ref) <= 1e-5 * m_ref
    want = update_bitfield(gr, float(mean.item()), cascades).reshape(cascades, -1)
    got = npy(bits).reshape(cascades, -1)
    for k in range(cascades):                                                                   # every max-pool level, given the mean
        assert np.array_equal(got[k], want[k]), f"cascade {k}"
    assert 0 < int(np.unpackbits(got[cascades - 1]).sum()) < G3                                 # the outermost cascade: a mixed pattern
    # a sparse grid: the max-pool must carry single occupied cells of cascade 0 outwards through every level
    sparse = np.zeros(n_el, np.float32)
    sparse[rng.integers(0, G3, 50)] = 1.0
    ops.grid_update_bitfield(cu(sparse), mean, bits, cascades)
    want = update_bitfield(sparse, float(mean.item()), cascades).reshape(cascades, -1)
    got = npy(bits).reshape(cascades, -1)
    assert np.array_equal(got, want) and all(int(np.count_nonzero(got[k])) > 0 for k in range(cascades))


# ------------------------------------------------------------------------------------------------ 11. hash table of wide scenes
def _march_ordered_coords(scenes, cascades, R=160):
    bits, _ = scenes[cascades]
    o, d = wide_rays(R, cascades, seed=30 + cascades)
    coords, _, _, cnt = oracle_march(o, d, bits, cascades, False, R * 1024)
    c = coords[:int(cnt[1])].copy()
    assert c.shape[0] > 3000 and c[:, :3].min() >= 0 and c[:, :3].max() <= 1 and np.ptp(c[:, :3], 0).min() > 0.5
    return c


@pytest.mark.parametrize("cascades", CASCADES)
def test_hash_and_fused_network_on_the_wide_scene_table(ops, scenes, cascades):
    """aabb_scale 64 (per_level_scale 1.823, finest resolution 131 072) and 32: level table, standalone hash forward and the fused
    forward / backward on march-ordered samples against the oracle chain (the chain of test_gpu_ops.test_network_bwd)."""
    aabb_scale = 1 << (cascades - 1)
    cfg = ol.HashCfg(aabb_scale)
    lv = ops.HashLevels(aabb_scale)
    assert np.array_equal(lv.offsets, cfg.offsets) and lv.per_level_scale == cfg.per_level_scale
    tab = npy(lv.table).view(np.uint32).reshape(16, 8)
    # The reference's grid_index forms its stride in 32 bits (HashEncode.h:77-91).  From resolution 65 536 on, resolution^2 wraps below
    # the level's size, the loop runs on and `hashmap_size < stride` is false: the finest level of these two tables is addressed by
    # x + y * res + z * (res^2 mod 2^32), not hashed.  Kernels and oracle keep that arithmetic, so a reference checkpoint means the same.
    def hashed(res, size):
        stride = 1
        for _ in range(3):
            if stride > size:
                break
            stride = (stride * res) & 0xFFFFFFFF
        return int(size < stride)
    assert [int(f) for f in tab[:, 4]] == [hashed(int(tab[l, 1]), int(tab[l, 3])) for l in range(16)] == [0] * 3 + [1] * 12 + [0]
    assert int(tab[15, 1]) in (2048 * aabb_scale, 2048 * aabb_scale + 1)                         # finest resolution (device exp2f: +-1 cell)
    coords = _march_ordered_coords(scenes, cascades)
    n = coords.shape[0]
    rng = np.random.default_rng(21)
    grid = rng.uniform(-1, 1, cfg.n_params).astype(np.float16)
    Wd, Wr = _mlp_weights(0, 3), _mlp_weights(1, 4)
    pos, dirs = coords[:, :3].copy(), coords[:, 4:].copy()
    enc = npy(ops.hash_fwd(cu(pos), cu(grid), lv))
    with device_scales(lv):
        enc_ref = ol.hash_fwd(cfg, pos, grid, acc32=True)
        out_ref, encr, hr = ol.network_fwd(cfg, pos, dirs, grid, Wd, Wr, acc32=True)
    assert np.abs(enc.astype(np.float32) - enc_ref.astype(np.float32)).max() <= 2e-3             # 1 fp16 ulp of O(1)
    out, enc_f = ops.network_fwd(cu(coords), cu(grid), lv, cu(Wd), cu(Wr))
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    assert np.abs(npy(enc_f).astype(np.float32) - encr.astype(np.float32)).max() <= 2e-3
    dd = np.abs(npy(out).astype(np.float32) - out_ref.astype(np.float32))
    assert dd.max() <= 2e-2 and dd.mean() <= 1e-3
    # backward
    dout = (rng.standard_normal((n, 4)) * 0.05).astype(np.float16)
    gg = torch.zeros(cfg.n_params, dtype=torch.float16, device="cuda")
    dwd = torch.zeros(Wd.size, dtype=torch.float32, device="cuda")
    dwr = torch.zeros(Wr.size, dtype=torch.float32, device="cuda")
    ops.network_bwd(cu(coords), enc_f, lv, cu(Wd), cu(Wr), cu(dout), gg, dwd, dwr)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    encr = npy(enc_f)                                            # start both chains from the same fp16 features
    h, inter_d = ol.mlp_fwd(Wd, encr, 0)
    rin = np.concatenate([h, ol.sh(dirs, np.float16)], 1)
    _, inter_r = ol.mlp_fwd(Wr, rin, 1)
    dYr = np.zeros((n, 16), np.float16)
    dYr[:, :3] = dout[:, :3]
    d_rin, _, dWr_ref = ol.mlp_bwd(Wr, rin, inter_r, dYr, 1, 3)
    dYd = d_rin[:, :16].astype(np.float32)
    dYd[:, 0] += dout[:, 3].astype(np.float32)
    d_enc, _, dWd_ref = ol.mlp_bwd(Wd, encr, inter_d, dYd.astype(np.float16), 0, 16)
    with device_scales(lv):
        gg_ref = ol.hash_bwd(cfg, pos, d_enc, acc32=True)
    sW = max(np.abs(dWr_ref).max(), np.abs(dWd_ref).max())
    assert np.abs(npy(dwr) - dWr_ref).max() <= 2e-2 * sW and np.abs(npy(dwd) - dWd_ref).max() <= 2e-2 * sW
    g = npy(gg).astype(np.float64)
    sG = np.abs(gg_ref).max()
    assert np.abs(g - gg_ref).max() <= 5e-2 * sG and np.abs(g - gg_ref).mean() <= 2e-3 * sG
    fine = slice(2 * int(cfg.offsets[15]), None)                 # the finest level (resolution 2048 * aabb_scale) received gradient
    assert np.count_nonzero(gg_ref[fine]) > 0 and np.count_nonzero(g[fine]) > 0


# ------------------------------------------------------------------------------------------------ llff_cfg on the stand-in
STAND_IN = dict(n_images=20, H=192, W=256, factor=2)              # loaded at 96 x 128: 17 training and 3 held-out views


def _llff_runner(root, seed, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.plugin.dataset import write_synthetic_llff
    from jnerf_b200.runner import Runner, llff_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    if not os.path.exists(os.path.join(root, "poses_bounds.npy")):
        write_synthetic_llff(root, seed=0, **STAND_IN)
    get_cfg().clear()
    update_cfg(**llff_cfg(root, seed=seed, **over))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].factor = STAND_IN["factor"]
    return Runner()


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """llff_cfg (7 cascades, cone stepping) trained for 1000 steps on the stand-in; also what it rendered before training."""
    root = str(tmp_path_factory.mktemp("llff"))
    r = _llff_runner(os.path.join(root, "fern"), seed=13, log_dir=os.path.join(root, "logs"))
    assert r.fast and r._fx is not None and r.sampler.NERF_CASCADES == 7 and r.sampler.const_dt is False      # the fused path
    psnr0 = r.psnr("val")
    r.train(steps=1000)
    torch.cuda.synchronize()
    return r, psnr0


def test_identical_ray_batch_to_radiance_at_seven_cascades(trained):
    """test_gpu_parity_e2e.py's chain on the trained LLFF state: one ray batch -> march -> fused network -> composite, CUDA against
    the oracle, with its bars."""
    from jnerf_b200 import ops
    r, _ = trained
    s, m, ds = r.sampler, r.model, r.dataset["train"]
    assert ds.aabb_scale == 64 and s.NERF_CASCADES == 7
    r._table_ready()
    r._sync_front()
    R = 384
    pix = ds.next_pixels(R)
    _, rays_o, rays_d = ds.rays_for(pix)
    rng = s.rng.copy()
    bits = s.density_grid_bitfield
    cap = R * 1024
    coords, ridx, numsteps, cnt = ops.march(rays_o.contiguous(), rays_d.contiguous(), bits, s.aabb_range, cap, s.cone_angle_constant,
                                            s.near_distance, s.NERF_CASCADES, s.const_dt, rng)
    S = int(cnt[1])
    assert S > 20 * R, S
    lv = m.pos_encoder.levels
    grid, Wd, Wr = m.pos_encoder.m_grid.detach(), m.density_mlp.con_weights.detach(), m.rgb_mlp.con_weights.detach()
    out, _ = ops.network_fwd(coords[:S].contiguous(), grid, lv, Wd, Wr)
    bg = torch.rand((R, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    ns_i = numsteps.view(torch.int32) if numsteps.dtype != torch.int32 else numsteps
    rgb = npy(ops.composite_fwd(out, coords[:S].contiguous(), ns_i, ns_i, bg, 7))
    rgb_i, alpha_i = ops.composite_infer(out, coords[:S].contiguous(), ns_i, 7)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    ref = ol.march(npy(rays_o), npy(rays_d), npy(bits), aabb=s.aabb_range, max_samples=cap, cone_angle=s.cone_angle_constant, near=s.near_distance,
                   cascades=7, const_dt=False, rng=np.asarray(rng, np.uint64))
    assert np.array_equal(npy(cnt).view(np.uint32), ref[3])
    assert np.array_equal(npy(numsteps).view(np.uint32), ref[2])
    assert np.array_equal(npy(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32))
    cfg = ol.HashCfg(64, log2_hashmap_size=19)
    assert cfg.n_params == grid.numel()
    c_np = ref[0][:S]
    with device_scales(lv):
        out_ref, _, _ = ol.network_fwd(cfg, c_np[:, :3].copy(), c_np[:, 4:].copy(), npy(grid).reshape(-1), npy(Wd).reshape(-1), npy(Wr).reshape(-1),
                                       acc32=True)
    rgb_ref = ol.composite_fwd(out_ref, c_np, ref[2], ref[2], npy(bg), 7)
    ri_ref, ai_ref = ol.composite_infer(out_ref, c_np, ref[2], 7)
    d_out = np.abs(npy(out).astype(np.float32) - out_ref.astype(np.float32))
    ulp = np.spacing(np.abs(out_ref).astype(np.float16)).astype(np.float32)
    err = np.abs(rgb - rgb_ref)
    stats = dict(samples=S, frac_bit_identical=float((d_out == 0).mean()), frac_within_2ulp=float((d_out <= 2 * ulp).mean()),
                 worst_excess=float((d_out - np.maximum(1e-2, 2 * ulp)).max()), rgb_max_abs=float(err.max()),
                 infer_rgb_max_abs=float(np.abs(npy(rgb_i) - ri_ref).max()), infer_alpha_max_abs=float(np.abs(npy(alpha_i) - ai_ref).max()))
    print("parity llff", stats)
    assert stats["frac_bit_identical"] > 0.80 and stats["frac_within_2ulp"] > 0.999 and stats["worst_excess"] <= 0, stats
    assert stats["rgb_max_abs"] <= 2e-4 and stats["infer_rgb_max_abs"] <= 2e-4 and stats["infer_alpha_max_abs"] <= 2e-4, stats


def test_llff_training_end_to_end(trained, tmp_path):
    """runner.llff_cfg on the stand-in at 96 x 128, 17 training views, 1000 steps.  Measured on an H100 80GB HBM3: held-out PSNR
    8.60 dB untrained -> 29.23 dB; the floor of 25 dB leaves margin."""
    from jnerf_b200 import ops
    r, psnr0 = trained
    s = r.sampler
    assert r.cfg.m_training_step == 1000 and ops.lib.load().ngp_debug_timeout_flag() == 0
    bits = s.density_grid_bitfield.reshape(7, -1)
    set_bits = [int(np.unpackbits(npy(bits[k])).sum()) for k in range(7)]
    print("llff occupancy bits per cascade", set_bits)
    assert 0 < set_bits[0] < G3 and sum(set_bits[1:]) > 0                                      # cascade 0 thinned out, outer cascades in use
    rng0 = s.rng.copy()
    psnr = r.test()                                                                           # the 3 held-out views, written as PNGs
    print("llff held-out psnr", psnr0, "->", psnr)
    assert psnr - psnr0 >= 6.0 and psnr >= PSNR_FLOOR, (psnr0, psnr)
    from PIL import Image
    test = r.dataset["test"]
    assert test.n_images == 3 and list(test.i_select) == [0, 8, 16]
    saved = np.asarray(Image.open(os.path.join(r.cfg.log_dir, r.cfg.exp_name, "test", f"{r.cfg.exp_name}_r_0.png")))
    s.rng[:] = rng0                                                                           # the jitter test() used for its first view
    img = r.render_img_with_pose(test.poses[0])
    u8 = (npy(img) * 255 + 0.5).clip(0, 255).astype(np.uint8)
    assert saved.shape == (96, 128, 3) and np.abs(u8.astype(np.int32) - saved.astype(np.int32)).max() <= 1
    for name in ("ckpt.pt", "params.pkl"):
        p = str(tmp_path / name)
        r.save_ckpt(p)
        table = r.model.pos_encoder.m_grid.detach().clone()
        r.model.pos_encoder.m_grid.data.zero_()
        s.density_grid_bitfield.zero_()
        r.load_ckpt(p)
        assert torch.equal(r.model.pos_encoder.m_grid.detach(), table) and int(s.density_grid_bitfield.count_nonzero()) > 0
        assert r.cfg.m_training_step == 1000
    assert torch.isfinite(r.train_step()).all()


PSNR_FLOOR = 25.0


def test_llff_training_is_deterministic(tmp_path):
    """Two seeded runs of 32 steps of llff_cfg (two occupancy-grid updates over 7 cascades each): bit-identical table and losses."""
    runs = []
    for _ in range(2):
        r = _llff_runner(str(tmp_path / "fern"), seed=5)
        losses = torch.stack([r.train_step().float().mean() for _ in range(32)])
        r._table_ready()
        torch.cuda.synchronize()
        runs.append((losses.cpu(), r.model.pos_encoder.m_grid.detach().clone(), r.sampler.density_grid_bitfield.clone(), r.sampler.n_rays_per_batch))
        del r
    a, b = runs
    assert torch.isfinite(a[0]).all() and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]
