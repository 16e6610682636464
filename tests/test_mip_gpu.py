"""The Mip-NeRF kernels (csrc/mip_sampler.cu, csrc/mip_mlp.cu) on the H100: ray generation against the reference's numpy, sampling and
resampling against an fp64 restatement given the same pcg32 uniforms, the fp32 encoder and the fused forward against the fp32 chain, the one
backward over both levels against autograd, the composite forward / loss backward against autograd, bit-identical seeded training, and
training on the lego stand-in on both network paths."""
import numpy as np
import pytest
import torch

import mip_cpu_backend as ref

pytestmark = pytest.mark.gpu

FWD_TOL = 12 * 2.0 ** -11          # as tests/test_nerf_gpu.py: eleven fp16 roundings after the shared encoding


def _cfg(using_fp16=True, seed=1, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.mip_runner import mip_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**mip_cfg(using_fp16=using_fp16, seed=seed, **over))
    return get_cfg()


def _rays(R, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    o = (torch.rand((R, 3), device="cuda", generator=g) - 0.5) * 8
    d = torch.nn.functional.normalize(-o + torch.randn((R, 3), device="cuda", generator=g) * 0.3, dim=-1) * (1 + torch.rand((R, 1), device="cuda", generator=g))
    rays = torch.cat([o, d, torch.nn.functional.normalize(d, dim=-1), torch.full((R, 1), 1.2e-3, device="cuda"), torch.full((R, 1), 2.0, device="cuda"),
                      torch.full((R, 1), 6.0, device="cuda")], -1)
    return rays.contiguous()


def test_rays_are_the_reference_numpy_bit_for_bit():
    from jnerf_b200 import ops
    from jnerf_b200.plugin.dataset import synthetic_cameras
    W, H, n = 40, 30, 3
    c2w = np.stack([np.asarray(m, np.float32)[:3, :4] for m in synthetic_cameras(n, seed=3)]).reshape(n, 12)
    images = torch.randint(0, 256, (n * H * W, 4), dtype=torch.uint8, device="cuda")
    pix = torch.randperm(n * H * W, device="cuda").int()
    rays, target = ops.mip_rays(pix, W, H, torch.from_numpy(c2w).cuda(), 51.3, 2.0, 6.0, images)
    want = ref.blender_rays_numpy(c2w, 51.3, W, H, 2.0, 6.0)[pix.cpu().long().numpy()]
    got = rays.cpu().numpy()
    assert np.array_equal(got, want), [(k, float(np.abs(got[:, k] - want[:, k]).max())) for k in range(12)]
    # the reference's img.astype(float32) / 255.0 (numpy: a correctly rounded division; torch's CUDA scalar division multiplies by 1/255)
    tar = images.cpu().numpy()[pix.cpu().long().numpy(), :3].astype(np.float32) / np.float32(255)
    assert np.array_equal(target.cpu().numpy(), tar)


@pytest.mark.parametrize("lindisp,randomized", [(False, True), (True, True), (False, False)])
def test_sample_and_resample_against_fp64(lindisp, randomized):
    from jnerf_b200 import ops
    R, S = 97, 128
    rays = _rays(R)
    rng = ops.pcg32_seed(11)
    t = ops.mip_sample(rays, S, lindisp, randomized, rng)
    u = torch.from_numpy(ref.pcg32_uniforms(rng, R, S + 1)).cuda()
    want = ref.sample(rays.double(), S, lindisp, randomized, u)
    assert (t.double() - want).abs().max().item() < 1e-5
    g = torch.Generator(device="cuda").manual_seed(2)
    w = torch.rand((R, S), device="cuda", generator=g) ** 8
    w[3] = 0                                                  # all-zero weights: the 1e-5 sum padding keeps the CDF defined
    w[5, 40:] = 0
    for padding, tol in ((0.01, 2e-4), (0.0, 4.0 / S)):
        # without padding, nearly empty intervals (w = rand^8) make the inverse CDF steep: an fp32 rounding of the CDF (~1e-7) moves a sample
        # by that over the local density, measured up to 0.0025 on the H100 for these weights; one interval width (4 / S) bounds it
        t2 = ops.mip_resample(t, w, padding, randomized, rng)
        want = ref.resample(t.double(), w.double(), padding, randomized, u)
        assert (t2.double() - want).abs().max().item() < tol, padding
        assert bool((t2[:, 1:] >= t2[:, :-1]).all()), "sorted"
        assert bool((t2 >= t[:, :1]).all() and (t2 <= t[:, -1:]).all())


def _chain(flat, enc, view):
    from jnerf_b200.plugin import mip
    p = mip.unpack(flat)
    lin = lambda name, x: x @ p[name][0].t() + p[name][1]
    h = enc
    for i in range(8):
        h = torch.relu(lin(f"layers.{i}.0", h))
        if i == 4:
            h = torch.cat([h, enc], -1)
    dens = lin("density_layer", h)
    v = torch.relu(lin("view_layers.0.0", torch.cat([lin("extra_layer", h), view], -1)))
    return torch.cat([lin("color_layer", v), dens], -1)


@pytest.mark.parametrize("ray_shape,integrate", [("cone", True), ("cylinder", True), ("cone", False)])
def test_encode_and_fused_forward_against_the_fp32_chain(ray_shape, integrate):
    from jnerf_b200 import ops
    from jnerf_b200.plugin import mip, nerf
    _cfg()
    P = mip.pack(nerf.init_reference_params(torch.Generator(device="cuda").manual_seed(4), mip.REF_LAYERS, mip.REF_ORDER))
    R, S = 37, 100                                            # 3700 rows: a partial last tile
    rays = _rays(R, seed=1)
    t = ops.mip_sample(rays, S, False, True, ops.pcg32_seed(3))
    enc, view = ops.mip_encode(rays, t, ray_shape, integrate, 0)
    e64, v64 = ref.encode(rays.double(), t.double(), ray_shape, integrate, 0, 8)
    assert (enc.double() - e64).abs().max().item() < 2e-4 and (view.double() - v64).abs().max().item() < 1e-5
    out = ops.mip_fwd(rays, t, P, ray_shape, integrate, 0)
    want = _chain(P, enc.half().float(), view.half().float())
    err = ((out.float() - want).abs() / (1 + want.abs())).max().item()
    assert torch.isfinite(out).all() and err <= FWD_TOL, err
    assert ops.mip_fwd(rays[:0], t[:0], P).shape == (0, 4)


def test_backward_over_both_levels_matches_autograd_and_is_deterministic():
    from jnerf_b200 import ops
    from jnerf_b200.plugin import mip, nerf
    _cfg()
    P = mip.pack(nerf.init_reference_params(torch.Generator(device="cuda").manual_seed(5), mip.REF_LAYERS, mip.REF_ORDER))
    R, S = 24, 128
    rays = _rays(R, seed=2)
    rng = ops.pcg32_seed(5)
    t_c = ops.mip_sample(rays, S, False, True, rng)
    t_f = ops.mip_sample(rays, S, True, True, rng)
    n = R * S
    half = ops.nerf_workspace_bytes(n)[0]
    saved = torch.empty(2 * half, dtype=torch.uint8, device="cuda")
    raw = torch.empty((2 * n, 4), dtype=torch.float16, device="cuda")
    ops.mip_fwd(rays, t_c, P, out=raw[:n], saved=saved[:half])
    ops.mip_fwd(rays, t_f, P, out=raw[n:], saved=saved[half:])
    dout = (torch.randn((2 * n, 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6)) * 0.1).half()
    grad = ops.nerf_bwd(P, saved, dout)
    assert torch.equal(grad, ops.nerf_bwd(P, saved, dout))
    leaves = {k: (W.clone().requires_grad_(), b.clone().requires_grad_()) for k, (W, b) in mip.unpack(P).items()}

    def chain(enc, view):
        lin = lambda name, x: x @ leaves[name][0].t() + leaves[name][1]
        h = enc
        for i in range(8):
            h = torch.relu(lin(f"layers.{i}.0", h))
            if i == 4:
                h = torch.cat([h, enc], -1)
        v = torch.relu(lin("view_layers.0.0", torch.cat([lin("extra_layer", h), view], -1)))
        return torch.cat([lin("color_layer", v), lin("density_layer", h)], -1)
    loss = 0
    for k, tt in enumerate((t_c, t_f)):
        enc, view = ops.mip_encode(rays, tt)
        loss = loss + (chain(enc.half().float(), view.half().float()) * dout[k * n:(k + 1) * n].float()).sum()
    loss.backward()
    got = mip.unpack(grad)
    rels = {}
    for name, (W, b) in leaves.items():
        for j, (tg, tr) in enumerate(((got[name][0], W.grad), (got[name][1], b.grad))):
            rels[name + (".weight", ".bias")[j]] = float((tg - tr).norm() / tr.norm().clamp_min(1e-12))
    print("relative gradient error per tensor:", {k: round(v, 4) for k, v in rels.items()})
    assert max(rels.values()) < 0.1, rels


@pytest.mark.parametrize("white,use_mask,cm,dtype", [(False, False, 0.1, torch.float32), (True, True, 0.5, torch.float32), (False, True, 0.1, torch.float16)])
def test_composite_forward_and_loss_backward_against_autograd(white, use_mask, cm, dtype):
    from jnerf_b200 import ops
    R, S = 53, 128
    rays = _rays(R, seed=4)
    rng = ops.pcg32_seed(9)
    t = torch.cat([ops.mip_sample(rays, S, False, True, rng), ops.mip_sample(rays, S, True, True, rng)])
    g = torch.Generator(device="cuda").manual_seed(8)
    raw = (torch.randn((2 * R * S, 4), device="cuda", generator=g) * 2).to(dtype)
    target = torch.rand((R, 3), device="cuda", generator=g)
    mask = (torch.rand(R, device="cuda", generator=g) > 0.3).float() if use_mask else None
    rgb, acc, dist, w = ops.mip_composite_fwd(raw[:R * S], t[:R], rays, 0.001, -1.0, white)
    c64 = ref.composite(raw[:R * S].double(), t[:R].double(), rays.double(), 0.001, -1.0, white)
    for got, want in ((rgb, c64[0]), (dist, c64[1]), (acc, c64[2]), (w, c64[3])):
        assert (got.double() - want).abs().max().item() < 1e-4
    scale = 100.0
    rgb2, loss, draw = ops.mip_composite_loss_bwd(raw, t, rays, target, mask, 0.001, -1.0, white, cm, grad_scale=scale)
    r64, l64, g64 = ref.loss_and_grad(raw.double(), t.double(), rays.double(), target.double(), mask, 0.001, -1.0, white, cm, scale)
    assert (rgb2.double() - r64).abs().max().item() < 1e-4 and abs(loss.double().sum().item() - l64.sum().item()) < 1e-5
    tol = 2e-3 if dtype == torch.float16 else 1e-5
    assert ((draw.double() - g64).abs() / (g64.abs().max() + 1e-12)).max().item() < tol


def _runner(using_fp16, seed, tmp_path, **over):
    from jnerf_b200.mip_runner import MipRunner
    cfg = _cfg(using_fp16, seed, log_dir=str(tmp_path), **over)
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=20, H=64, W=64, batch_size=cfg.dataset[split].batch_size if split == "train" else 64)
    return MipRunner()


def test_two_seeded_runs_are_bit_identical(tmp_path):
    params = []
    for _ in range(2):
        r = _runner(True, 3, tmp_path)
        r.train(20)
        torch.cuda.synchronize()
        params.append(r.model.params.detach().clone())
    assert torch.equal(params[0], params[1])
    assert not torch.equal(params[0], _runner(True, 3, tmp_path).model.params.detach())


STEPS = 400
# mip_base.py's 2500-step warm-up at 1 % of the rate and its 288-ray batches learn too little in a test's budget: a short schedule
SCHED = dict(optim=dict(type="Adam", lr=2e-3, eps=1e-15, betas=(0.9, 0.99)),
             linearlog=dict(type="LinearLog", end_lr=2e-4, max_steps=STEPS, lr_delay_steps=0, lr_delay_mult=1.0))


def test_training_both_paths_on_the_lego_stand_in(tmp_path):
    res = {}
    for fp16 in (True, False):
        r = _runner(fp16, 5, tmp_path / str(fp16), **SCHED)
        r.cfg.dataset.train.batch_size = 1024
        r.dataset["train"].batch_size = 1024
        p0 = r.test()
        r.train(STEPS)
        p1 = r.test()
        res[fp16] = (p0, p1)
        out = tmp_path / str(fp16) / "lego_sss" / "test"
        assert sorted(p.name for p in out.iterdir()) == ["lego_sss_gt_0.png", "lego_sss_gt_1.png", "lego_sss_r_0.png", "lego_sss_r_1.png"]
    print(f"mip_cfg lego stand-in, {STEPS} steps: fused fp16 {res[True][0]:.2f} -> {res[True][1]:.2f} dB, "
          f"fp32 chain {res[False][0]:.2f} -> {res[False][1]:.2f} dB")
    for p0, p1 in res.values():
        assert p1 > p0 + 5.0, res
    assert abs(res[True][1] - res[False][1]) < 0.5, res
