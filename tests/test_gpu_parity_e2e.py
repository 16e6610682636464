"""Parity at the level north_star states it: identical ray batch -> march -> fused network -> composite, CUDA path against
the oracle chain, on BASELINE config #2 (lego settings: aabb 1, const_dt, T=2^19) and config #3 (fox settings: aabb 4, cone
stepping, ngp_fox.py:68-73) with a TRAINED state (table, weights and occupancy bitfield after a few hundred steps), plus the
independent check of the fully-fused MLP against the reference's own other definition of the same network -- the plain
Linear/ReLU chain of models/networks/ngp_network.py:59-67 -- evaluated by PyTorch in fp32 with autograd.

Bars: sample indices / step counts / coordinates bit-exact; radiance within 1e-3 (absolute on [0,1] radiance = relative to full
scale, and relative to the pixel for pixels brighter than 0.1)."""
import numpy as np
import pytest
import torch

import oracle_lib as ol
from test_gpu_ops import cu, device_scales, npy

pytestmark = pytest.mark.gpu


def _trained_runner(kind, steps):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    if kind == "lego":
        update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=13))
        cfg = get_cfg()
        cfg.dataset.train.n_images = 8
        cfg.dataset.train.H = cfg.dataset.train.W = 160
        cfg.dataset.val = None
    else:
        update_cfg(**fox_cfg(fp16=True, synthetic=True, seed=13))
        cfg = get_cfg()
        cfg.dataset.train.n_images = 8
        cfg.dataset.train.W, cfg.dataset.train.H = 90, 160
    r = Runner()
    for _ in range(steps):
        r.train_step()
    torch.cuda.synchronize()
    return r


@pytest.mark.parametrize("kind", ["lego", "fox"])
def test_identical_ray_batch_to_radiance(kind):
    from jnerf_b200 import ops
    r = _trained_runner(kind, 300)
    s, m, ds = r.sampler, r.model, r.dataset["train"]
    aabb_scale = 1 if kind == "lego" else 4
    assert ds.aabb_scale == aabb_scale and s.const_dt == (kind == "lego")
    R = 384
    pix = ds.next_pixels(R)
    _, rays_o, rays_d = ds.rays_for(pix)
    rng = s.rng.copy()
    bits = s.density_grid_bitfield
    assert int(bits.count_nonzero()) > 0
    cap = R * 1024
    # ---------------- CUDA path through the C ABI
    coords, ridx, numsteps, cnt = ops.march(rays_o.contiguous(), rays_d.contiguous(), bits, s.aabb_range, cap, s.cone_angle_constant,
                                            s.near_distance, s.NERF_CASCADES, s.const_dt, rng)
    S = int(cnt[1])
    assert S > 20 * R, S                                             # the trained scene really is sampled
    lv = m.pos_encoder.levels
    grid, Wd, Wr = m.pos_encoder.m_grid.detach(), m.density_mlp.con_weights.detach(), m.rgb_mlp.con_weights.detach()
    out, _ = ops.network_fwd(coords[:S].contiguous(), grid, lv, Wd, Wr)
    bg = torch.rand((R, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    ns_i = numsteps.view(torch.int32) if numsteps.dtype != torch.int32 else numsteps
    rgb = npy(ops.composite_fwd(out, coords[:S].contiguous(), ns_i, ns_i, bg))
    rgb_i, alpha_i = ops.composite_infer(out, coords[:S].contiguous(), ns_i)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    # ---------------- oracle chain on the same inputs
    o_np, d_np = npy(rays_o), npy(rays_d)
    ref = ol.march(o_np, d_np, npy(bits), aabb=s.aabb_range, max_samples=cap, cone_angle=s.cone_angle_constant, near=s.near_distance,
                   cascades=s.NERF_CASCADES, const_dt=s.const_dt, rng=np.asarray(rng, np.uint64))
    assert np.array_equal(npy(cnt).view(np.uint32), ref[3])
    assert np.array_equal(npy(numsteps).view(np.uint32), ref[2])                           # sample counts and bases: bit-exact
    assert np.array_equal(npy(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32))     # every sample: bit-exact
    cfg = ol.HashCfg(aabb_scale, log2_hashmap_size=19)
    assert cfg.n_params == grid.numel()
    c_np = ref[0][:S]
    with device_scales(lv):
        out_ref, _, _ = ol.network_fwd(cfg, c_np[:, :3].copy(), c_np[:, 4:].copy(), npy(grid).reshape(-1), npy(Wd).reshape(-1),
                                       npy(Wr).reshape(-1), acc32=True)
    rgb_ref = ol.composite_fwd(out_ref, c_np, ref[2], ref[2], npy(bg))
    ri_ref, ai_ref = ol.composite_infer(out_ref, c_np, ref[2])
    # per-sample network output (fp16): the two paths round the same fp32 dot products, accumulated in a different order, to fp16 at
    # every layer; they agree bit for bit except where a sum lands on a rounding boundary
    d_out = np.abs(npy(out).astype(np.float32) - out_ref.astype(np.float32))
    ulp = np.spacing(np.abs(out_ref).astype(np.float16)).astype(np.float32)
    err = np.abs(rgb - rgb_ref)
    bright = rgb_ref > 0.1
    stats = dict(samples=S, frac_bit_identical=float((d_out == 0).mean()), frac_within_2ulp=float((d_out <= 2 * ulp).mean()),
                 worst_excess=float((d_out - np.maximum(1e-2, 2 * ulp)).max()),
                 out_max_abs=float(d_out.max()), out_absmax_ref=float(np.abs(out_ref).max()), rgb_max_abs=float(err.max()), rgb_mean_abs=float(err.mean()),
                 rgb_max_rel_bright=float((err[bright] / rgb_ref[bright]).max()) if bright.any() else 0.0,
                 infer_rgb_max_abs=float(np.abs(npy(rgb_i) - ri_ref).max()), infer_alpha_max_abs=float(np.abs(npy(alpha_i) - ai_ref).max()))
    print("parity", kind, stats)
    # per sample: bit-identical for the bulk, within 2 fp16 ulp for 99.9 %; the tail is a hidden activation that rounded the other way
    # (1 ulp of an O(1..8) activation times an O(0.3) weight), bounded absolutely
    # (1e-2, or 2 ulp where the output itself is large: the fox scene's raw densities reach +-25, where one fp16 ulp is 0.0156)
    assert stats["frac_bit_identical"] > 0.80 and stats["frac_within_2ulp"] > 0.999 and stats["worst_excess"] <= 0, stats
    # radiance: north_star's bar is 1e-3 (absolute on [0,1] radiance, and relative to the pixel for pixels brighter than 0.1);
    # asserted at 2e-4 so that a regression shows long before the 1e-3 bar is at risk
    assert stats["rgb_max_abs"] <= 2e-4 and stats["rgb_max_rel_bright"] <= 2e-4, stats
    assert stats["infer_rgb_max_abs"] <= 2e-4 and stats["infer_alpha_max_abs"] <= 2e-4, stats


# --------------------------------------------------------------------------------------------- MLP vs torch fp32 Linear/ReLU
def _torch_chain(Ws, x, round_fp16):
    """ngp_network.py:59-67: Linear(bias=False) / ReLU chain.  round_fp16: activations stored as fp16 between layers (what the
    fp16 nn.Linear path does: every layer's output tensor is float16); the matmuls themselves run in fp32."""
    h = x
    for k, W in enumerate(Ws):
        h = h @ W.t()
        if k + 1 < len(Ws):
            h = torch.relu(h)
        if round_fp16:
            h = h.half().float()
    return h


def _split(W, nhm):
    shapes = [(64, 32)] + [(64, 64)] * nhm + [(16, 64)]
    out, off = [], 0
    for s in shapes:
        out.append(W[off:off + s[0] * s[1]].reshape(s))
        off += s[0] * s[1]
    return out


@pytest.mark.parametrize("nhm,n_valid", [(0, 16), (1, 3)])
def test_mlp_against_torch_fp32_linear_chain_with_autograd(nhm, n_valid):
    """ngp_mlp_fwd / ngp_mlp_bwd against a plain PyTorch fp32 Linear/ReLU chain + autograd (no oracle involved)."""
    from jnerf_b200 import ops
    from test_gpu_ops import _mlp_weights
    torch.backends.cuda.matmul.allow_tf32 = False
    n = 8192
    g = torch.Generator(device="cuda").manual_seed(17)
    W = cu(_mlp_weights(nhm, 2))
    X = torch.randn((n, 32), device="cuda", generator=g).clamp(-4, 4).half()
    dY = (torch.randn((n, 16), device="cuda", generator=g) * 0.1).half()
    dY[:, n_valid:] = 0
    Y, inter = ops.mlp_fwd(W, X, nhm)
    Ws = [w.float().requires_grad_(True) for w in _split(W, nhm)]
    Xf = X.float().requires_grad_(True)
    Yt = _torch_chain(Ws, Xf, round_fp16=True)
    # forward: same fp16 rounding points, fp32 accumulation in another order -> bit-identical except at rounding boundaries
    d = (Y.float() - Yt.detach()).abs()
    ulp = torch.from_numpy(np.spacing(np.abs(npy(Yt.detach())).astype(np.float16)).astype(np.float32)).cuda()
    assert float((d == 0).float().mean()) > 0.9 and float((d <= 2 * ulp).float().mean()) > 0.999 and float((d / ulp.clamp_min(2.0 ** -14)).max()) <= 8
    # and against the chain with NO intermediate rounding (pure fp32 network): fp16 storage error of a 2-3 layer net, 1e-3 relative
    Y32 = _torch_chain([w.detach() for w in Ws], X.float(), round_fp16=False)
    assert float((Y.float() - Y32).abs().max()) <= 4e-3 * float(Y32.abs().max())
    Yt.backward(dY.float())
    dX, _, dW = ops.mlp_bwd(W, X, inter, dY, nhm, n_valid, need_dx=True, need_temps=False)
    dWt = torch.cat([w.grad.reshape(-1) for w in Ws])
    sW = float(dWt.abs().max())
    # weight gradients: sums over 8192 rows of fp16 x fp16 products, fp32 accumulation on both sides
    assert float((dW - dWt).abs().max()) <= 1e-3 * sW, (float((dW - dWt).abs().max()), sW)
    off = 64 * 32 + nhm * 64 * 64
    assert (dW[off + n_valid * 64:] == 0).all()
    sX = float(Xf.grad.abs().max())
    assert float((dX.float() - Xf.grad).abs().max()) <= 2e-3 * sX


@pytest.mark.parametrize("aabb,log2T", [(1, 19), (4, 19)])
def test_fused_network_against_torch_composition(aabb, log2T):
    """The fused forward / backward kernels against the per-operator composition the reference itself falls back to on a GPU its
    binary does not support (ngp_network.py:59-67,77-84): HashEncoder (ngp_hash_fwd, pinned to the reference sources) -> torch fp32
    Linear/ReLU chains -> autograd -> ngp_hash_bwd.  Production table size, lego (aabb 1) and fox (aabb 4) level tables."""
    from jnerf_b200 import ops
    from test_gpu_ops import _mlp_weights
    torch.backends.cuda.matmul.allow_tf32 = False
    n = 16384
    lv = ops.HashLevels(aabb, log2_hashmap_size=log2T)
    g = torch.Generator(device="cuda").manual_seed(23)
    coords = torch.zeros((n, 7), device="cuda")
    # ray-ordered-like positions: short runs along random segments, so that run-length combining in the scatter is exercised
    n_seg = n // 64
    a = torch.rand((n_seg, 1, 3), device="cuda", generator=g)
    b = torch.rand((n_seg, 1, 3), device="cuda", generator=g)
    t = torch.linspace(0, 1, 64, device="cuda").view(1, 64, 1)
    coords[:, :3] = (a + (b - a) * t * 0.2).clamp(0, 1).reshape(n, 3)
    coords[:, 4:] = torch.rand((n, 3), device="cuda", generator=g)
    n_params = int(lv.offsets[-1]) * 2
    grid = (torch.rand(n_params, device="cuda", generator=g) * 2 - 1).half()
    Wd, Wr = cu(_mlp_weights(0, 3)), cu(_mlp_weights(1, 4))
    dout = (torch.randn((n, 4), device="cuda", generator=g) * 0.05).half()
    out, enc = ops.network_fwd(coords, grid, lv, Wd, Wr)
    gg = torch.zeros(n_params, dtype=torch.float16, device="cuda")
    dwd, dwr = torch.zeros(3072, device="cuda"), torch.zeros(7168, device="cuda")
    ops.network_bwd(coords, enc, lv, Wd, Wr, dout, gg, dwd, dwr)
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    # composition
    enc_t = ops.hash_fwd(coords[:, :3].contiguous(), grid, lv)
    assert float((enc.float() - enc_t.float()).abs().max()) <= 2e-3            # fused gather == standalone HashEncoder (1 fp16 ulp of O(1))
    sh = ops.sh_fwd(coords[:, 4:].contiguous(), torch.float16)
    Wds = [w.float().requires_grad_(True) for w in _split(Wd, 0)]
    Wrs = [w.float().requires_grad_(True) for w in _split(Wr, 1)]
    e = enc.float().requires_grad_(True)                                       # both chains start from the same fp16 features
    h = _torch_chain(Wds, e, round_fp16=True)                                  # (n,16): column 0 = raw density
    rgb = _torch_chain(Wrs, torch.cat([h, sh.float()], 1), round_fp16=True)    # (n,16): columns 0..2
    out_t = torch.cat([rgb[:, :3], h[:, :1]], 1)
    d = (out.float() - out_t.detach()).abs()
    ulp = torch.from_numpy(np.spacing(np.abs(npy(out_t.detach())).astype(np.float16)).astype(np.float32)).cuda()
    assert float((d == 0).float().mean()) > 0.8 and float((d <= 2 * ulp).float().mean()) > 0.995 and float((d / ulp.clamp_min(2.0 ** -14)).max()) <= 16
    out_t.backward(dout.float())
    dWd_t = torch.cat([w.grad.reshape(-1) for w in Wds])
    dWr_t = torch.cat([w.grad.reshape(-1) for w in Wrs])
    # weight gradients: 16 384-row sums of fp16 x fp16 products, fp32 accumulation on both sides; the addends differ where an fp16
    # gradient slab entry rounded the other way (1 ulp = 2^-11 relative of one addend) -- measured 2.5e-3 of the largest entry
    assert float((dwd - dWd_t).abs().max()) <= 5e-3 * float(dWd_t.abs().max())
    assert float((dwr - dWr_t).abs().max()) <= 5e-3 * float(dWr_t.abs().max())
    gg_t = ops.hash_bwd(coords[:, :3].contiguous(), e.grad.half().contiguous(), lv).float()
    sG = float(gg_t.abs().max())
    dg = (gg.float() - gg_t).abs()
    # both sides sum fp16-rounded addends with f16x2 reductions in a nondeterministic order (HashEncode.h:339-347 does the same); the
    # fused kernel pre-reduces runs in fp32 (fewer roundings).  Every reduction rounds the running sum to fp16 (2^-11 relative), so an
    # entry that receives n addends carries up to n x 2^-11 of its magnitude: ~1e-2 of the largest entry for the busiest coarse-level
    # entries (measured 1.3e-2 on the fox table), 3e-7 on average.
    assert float(dg.max()) <= 2e-2 * sG and float(dg.mean()) <= 2e-4 * sG, (float(dg.max()), float(dg.mean()), sG)
