"""multicam.py's Mip-NeRF on the H100 (csrc/mip_multiscale.cu, csrc/mip_mlp_wide.cu): the rays, targets and loss weights of Blenders and
Multicam against the reference's numpy (tests/multicam_cpu_backend.py), the 16-degree fp32 encoder against fp64 with a per-degree bound, the
96-wide fused network against the fp32 chain and autograd, bit-identical seeded runs, and training on the multiscale stand-in on both network
paths with the per-resolution test PSNR."""
import math

import numpy as np
import pytest
import torch

import mip_cpu_backend as ref
import multicam_cpu_backend as mref
import nerf_mlp_ref
from test_mip_gpu import FWD_TOL

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -23


def _check_rays(ds, images, white):
    want_r, want_t, want_m = mref.nerf_py_rays(images, ds.table["cams"].cpu().numpy(), ds.focal, white)
    pix = torch.randperm(ds.offsets[-1], device="cuda").int()
    rays, target, lossmult = ds.rays_for(pix)
    idx = pix.cpu().long().numpy()
    want_r, want_t, want_m = want_r[idx], want_t[idx], want_m[idx]
    got = rays.cpu().numpy()
    # targets, loss weights, origins, near and far bit for bit; the reference's @ runs through BLAS (Multicam) or in fp64 (Blenders, whose
    # fp64 focal length promotes numpy to fp64): directions and viewdirs within 8 fp32 ulps of the largest component, radii within 16 ulps of it (a difference of
    # two directions) times 2 / sqrt(12)
    assert np.array_equal(target.cpu().numpy(), want_t) and np.array_equal(lossmult.cpu().numpy(), want_m)
    assert np.array_equal(got[:, [0, 1, 2, 10, 11]], want_r[:, [0, 1, 2, 10, 11]])
    dmax = np.abs(want_r[:, 3:6]).max(-1, keepdims=True)
    assert (np.abs(got[:, 3:6] - want_r[:, 3:6]) <= 8 * EPS * dmax).all()
    assert (np.abs(got[:, 6:9] - want_r[:, 6:9]) <= 8 * EPS).all()
    err = np.abs(got[:, 9] - want_r[:, 9]) / (16 * EPS * dmax[:, 0] * 2 / math.sqrt(12))
    assert err.max() <= 1.0, err.max()
    return err.max()


def test_multiscale_rays_and_targets_against_the_reference_numpy(tmp_path):
    from jnerf_b200.plugin import dataset as D, mip
    root = str(tmp_path / "lego")
    D.write_synthetic_multicam(root, n_images=6, H=64, W=48, seed=4)
    for white in (True, False):
        mc = mip.Multicam(root, "train", white_bkgd=white)
        flat = mc.table["images"].cpu().numpy()
        images = [flat[mc.offsets[i]:mc.offsets[i + 1]].reshape(mc.Hs[i], mc.Ws[i], 4) for i in range(mc.n_images)]
        print("Multicam radius error / bound:", _check_rays(mc, images, white))
        for factor in (0, 2):
            bl = mip.Blenders(root, "train", white_bkgd=white, factor=factor)
            flat = bl.table["images"].cpu().numpy()
            images = [flat[bl.offsets[i]:bl.offsets[i + 1]].reshape(bl.H, bl.W, 4) for i in range(bl.n_images)]
            print(f"Blenders factor {factor} radius error / bound:", _check_rays(bl, images, white))


def _rays(R, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    o = (torch.rand((R, 3), device="cuda", generator=g) - 0.5) * 8
    d = torch.nn.functional.normalize(-o + torch.randn((R, 3), device="cuda", generator=g) * 0.3, dim=-1) * (1 + torch.rand((R, 1), device="cuda", generator=g))
    return torch.cat([o, d, torch.nn.functional.normalize(d, dim=-1), torch.full((R, 1), 1.2e-3, device="cuda"), torch.full((R, 1), 2.0, device="cuda"),
                      torch.full((R, 1), 6.0, device="cuda")], -1).contiguous()


@pytest.mark.parametrize("ray_shape,integrate", [("cone", True), ("cylinder", True), ("cone", False)])
def test_16_degree_encoder_against_fp64_per_degree(ray_shape, integrate):
    """Column (k, dim) of degree k against float64, within the per-degree bound of tests/nerf_mlp_ref.py: ipe64."""
    from jnerf_b200 import ops
    R, S = 61, 128
    rays = _rays(R, seed=3)
    t = ops.mip_sample(rays, S, False, True, ops.pcg32_seed(7))
    enc, view = ops.mip_encode(rays, t, ray_shape, integrate, 0, degs=16)
    assert enc.shape == (R * S, 96)
    want, bound = nerf_mlp_ref.ipe64(rays, t, ray_shape, integrate, 16)
    ratio = ((enc.double() - want).abs() / bound).reshape(-1, 2, 16, 3).amax((0, 1, 3))
    print(f"{ray_shape} integrate={integrate}: worst error / bound per degree", [round(float(x), 3) for x in ratio])
    assert float(ratio.max()) <= 1.0
    _, v64 = ref.encode(rays.double(), t.double(), ray_shape, integrate, 0, 8)
    assert (view.double() - v64).abs().max().item() < 1e-5
    # the new entry point at 8 degrees is the existing encoder bit for bit
    e8, v8 = ops.mip_encode(rays, t, ray_shape, integrate, 0)
    from jnerf_b200 import lib
    e8b, v8b = torch.empty_like(e8), torch.empty_like(v8)
    lib.call("ngp_mip_encode_deg", ops._stream(), R, S, ops._p(rays), ops._p(t), ops.RAY_SHAPES.index(ray_shape), int(integrate), 0, 8,
             ops._p(e8b), ops._p(v8b))
    assert torch.equal(e8, e8b) and torch.equal(v8, v8b)
    assert torch.equal(enc[:, :24], e8[:, :24]) and torch.equal(enc[:, 48:72], e8[:, 24:])     # degrees 0..7 are the 8-degree columns


def _wide_params(seed):
    from jnerf_b200.plugin import mip, nerf
    return mip.pack(nerf.init_reference_params(torch.Generator(device="cuda").manual_seed(seed), mip.ref_layers(16), mip.REF_ORDER), 16)


def _chain16(leaves, enc, view):
    lin = lambda name, x: x @ leaves[name][0].t() + leaves[name][1]
    h = enc
    for i in range(8):
        h = torch.relu(lin(f"layers.{i}.0", h))
        if i == 4:
            h = torch.cat([h, enc], -1)
    v = torch.relu(lin("view_layers.0.0", torch.cat([lin("extra_layer", h), view], -1)))
    return torch.cat([lin("color_layer", v), lin("density_layer", h)], -1)


def _saved_encoding(saved, n):
    """The 12 encoding groups of the fused forward's saved blocks (320 groups of [128 rows][8 halfs] a tile) as (n, 96) fp16."""
    T = (n + 127) // 128
    blocks = saved[:T * 320 * 128 * 16].view(torch.float16).view(T, 320, 128, 8)[:, :12]
    return blocks.permute(0, 2, 1, 3).reshape(T * 128, 96)[:n]


@pytest.mark.parametrize("ray_shape,integrate", [("cone", True), ("cylinder", True), ("cone", False)])
def test_wide_fused_forward_against_the_fp32_chain(ray_shape, integrate):
    """The 96-wide fused forward: its saved encoding is mip_encode(..., degs=16).half() bit for bit, its outputs are the fp32 chain's on
    those encodings within test_mip_gpu.py's FWD_TOL, on 3700 rows (a partial last tile)."""
    from jnerf_b200 import ops
    from jnerf_b200.plugin import mip
    assert ops.mip_param_count(16) == 618912 and ops.mip_param_count(8) == ops.nerf_param_count()
    P = _wide_params(4)
    R, S = 37, 100
    rays = _rays(R, seed=1)
    t = ops.mip_sample(rays, S, False, True, ops.pcg32_seed(3))
    enc, view = ops.mip_encode(rays, t, ray_shape, integrate, 0, degs=16)
    n = R * S
    saved = torch.empty(ops.mip_workspace_bytes(n, 16)[0], dtype=torch.uint8, device="cuda")
    out = ops.mip_fwd(rays, t, P, ray_shape, integrate, 0, saved=saved, degs=16)
    assert torch.equal(_saved_encoding(saved, n).view(torch.int16), enc.half().view(torch.int16))
    assert torch.equal(out, ops.mip_fwd(rays, t, P, ray_shape, integrate, 0, degs=16))
    want = _chain16(mip.unpack(P, 16), enc.half().float(), view.half().float())
    err = ((out.float() - want).abs() / (1 + want.abs())).max().item()
    print(f"{ray_shape} integrate={integrate}: 96-wide forward error {err:.2e} (FWD_TOL {FWD_TOL:.2e})")
    assert torch.isfinite(out).all() and err <= FWD_TOL, err
    assert ops.mip_fwd(rays[:0], t[:0], P, degs=16).shape == (0, 4)


def test_wide_backward_over_both_levels_matches_autograd_and_is_deterministic():
    from jnerf_b200 import ops
    from jnerf_b200.plugin import mip
    P = _wide_params(5)
    R, S = 24, 128
    rays = _rays(R, seed=2)
    rng = ops.pcg32_seed(5)
    t_c = ops.mip_sample(rays, S, False, True, rng)
    t_f = ops.mip_sample(rays, S, True, True, rng)
    n = R * S
    half = ops.mip_workspace_bytes(n, 16)[0]
    saved = torch.empty(2 * half, dtype=torch.uint8, device="cuda")
    raw = torch.empty((2 * n, 4), dtype=torch.float16, device="cuda")
    ops.mip_fwd(rays, t_c, P, out=raw[:n], saved=saved[:half], degs=16)
    ops.mip_fwd(rays, t_f, P, out=raw[n:], saved=saved[half:], degs=16)
    dout = (torch.randn((2 * n, 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6)) * 0.1).half()
    grad = ops.mip_bwd(P, saved, dout, 16)
    assert grad.shape == (618912,) and torch.equal(grad, ops.mip_bwd(P, saved, dout, 16))
    leaves = {k: (W.clone().requires_grad_(), b.clone().requires_grad_()) for k, (W, b) in mip.unpack(P, 16).items()}
    loss = 0
    for k, tt in enumerate((t_c, t_f)):
        enc, view = ops.mip_encode(rays, tt, degs=16)
        loss = loss + (_chain16(leaves, enc.half().float(), view.half().float()) * dout[k * n:(k + 1) * n].float()).sum()
    loss.backward()
    got = mip.unpack(grad, 16)
    rels = {}
    for name, (W, b) in leaves.items():
        for j, (tg, tr) in enumerate(((got[name][0], W.grad), (got[name][1], b.grad))):
            rels[name + (".weight", ".bias")[j]] = float((tg - tr).norm() / tr.norm().clamp_min(1e-12))
    print("96-wide relative gradient error per tensor:", {k: round(v, 4) for k, v in rels.items()})
    assert max(rels.values()) < 0.1, rels
    # padding stays zero: no gradient reaches a parameter outside the reference's tensors
    mask = mip.pack({k: (torch.ones_like(W), torch.ones_like(b)) for k, (W, b) in leaves.items()}, 16) != 0
    assert not grad[~mask].any()


def _multicam_runner(tmp_path, using_fp16, seed, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.mip_runner import MipRunner, multicam_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**multicam_cfg(seed=seed, log_dir=str(tmp_path), using_fp16=using_fp16, **over))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=20, H=64, W=64)
    cfg.dataset.train.batch_size = 1024
    return MipRunner()


def test_two_seeded_fused_multicam_runs_are_bit_identical(tmp_path):
    params = []
    for _ in range(2):
        r = _multicam_runner(tmp_path, True, 3)
        assert r.model.params.numel() == 618912
        r.train(20)
        torch.cuda.synchronize()
        params.append(r.model.params.detach().clone())
    assert torch.equal(params[0], params[1])
    assert not torch.equal(params[0], _multicam_runner(tmp_path, True, 3).model.params.detach())


STEPS = 400
SCHED = dict(optim=dict(type="Adam", lr=2e-3, eps=1e-15, betas=(0.9, 0.99)),
             linearlog=dict(type="LinearLog", end_lr=2e-4, max_steps=STEPS, lr_delay_steps=0, lr_delay_mult=1.0))


def test_training_on_the_multiscale_stand_in(tmp_path, capsys):
    """multicam_cfg (16 degrees) on the in-memory multiscale stand-in, fused fp16 and fp32 chain: the test PSNR of every resolution rises by
    > 5 dB, and the two paths end within 0.5 dB of each other at every resolution."""
    res = {}
    for fp16 in (True, False):
        r = _multicam_runner(tmp_path / str(fp16), fp16, 5, **SCHED)
        r.test()
        p0 = dict(r.test_psnr_by_size)
        r.train(STEPS)
        r.test()
        res[fp16] = (p0, dict(r.test_psnr_by_size))
    with capsys.disabled():
        for fp16, (p0, p1) in res.items():
            print(f"\nmulticam_cfg multiscale stand-in (64x64 full res), {'fused fp16' if fp16 else 'fp32 chain'}, 16 degrees, {STEPS} steps of "
                  "1024 rays, test PSNR:", {f"{w}x{h}": f"{p0[(w, h)]:.2f} -> {p1[(w, h)]:.2f} dB" for (w, h) in p1})
    for p0, p1 in res.values():
        assert sorted(p1) == [(8, 8), (16, 16), (32, 32), (64, 64)]
        for key in p1:
            assert p1[key] > p0[key] + 5.0, (key, p0, p1)
    for key in res[True][1]:
        assert abs(res[True][1][key] - res[False][1][key]) < 0.5, (key, res)
