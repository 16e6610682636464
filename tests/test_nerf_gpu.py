"""The vanilla NeRF kernels (csrc/nerf_mlp.cu) on the H100: the fused forward against the fp32 torch chain on the same fp16 weights and
encodings (partial tiles, N = 0, a device row count below N), the density kernel against the forward's alpha column bit for bit, the
deterministic backward against torch autograd, training of nerf_cfg on the lego stand-in against the fp32 path, and the whole-frame
renderer against render_img."""
import numpy as np
import pytest
import torch

import nerf_mlp_ref

pytestmark = pytest.mark.gpu

# Every activation is rounded to fp16 once (relative error <= 2^-11) and the chain has 11 roundings after the shared encoding; with the
# near-unit gain of the initialised layers the output error stays within a few multiples of that.  12 x 2^-11 of (1 + |ref|) bounds it.
FWD_TOL = 12 * 2.0 ** -11


def _setup(fp16=True, seed=1):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import nerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**nerf_cfg(fp16=fp16, synthetic=True, seed=seed))
    from jnerf_b200.plugin import nerf
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return nerf, nerf.pack(nerf.init_reference_params(gen))


def _coords(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.rand((n, 7), device="cuda", generator=g)
    c[:, 3] = 0
    return c


def _torch_chain(nerf, ref, coords):
    """ori_nerf_network.py:34-56 in fp32 on the fp16-rounded encodings; ref = {name: (W, b)} fp32 leaves."""
    enc = nerf.freq_encode(coords[:, :3], 10).half().float()
    encd = nerf.freq_encode(coords[:, 4:7], 4).half().float()
    lin = lambda name, x: x @ ref[name][0].t() + ref[name][1]
    h = enc
    for i in range(8):
        h = torch.relu(lin(f"pts_linears.{i}", h))
        if i == 4:
            h = torch.cat([enc, h], -1)
    alpha = lin("alpha_linear", h)
    v = torch.relu(lin("views_linears.0", torch.cat([lin("feature_linear", h), encd], -1)))
    return torch.cat([lin("rgb_linear", v), alpha], -1)


@pytest.mark.parametrize("n", [1000, 128 * 37, 1])
def test_forward_matches_fp32_chain(n):
    from jnerf_b200 import ops
    nerf, P = _setup()
    c = _coords(n)
    out, _ = ops.nerf_fwd(c, P)
    ref = _torch_chain(nerf, nerf.unpack(P), c)
    err = (out.float() - ref).abs()
    assert torch.isfinite(out).all()
    assert float((err / (1 + ref.abs())).max()) <= FWD_TOL, float(err.max())


def test_forward_empty_and_device_row_count():
    from jnerf_b200 import ops
    nerf, P = _setup()
    out, _ = ops.nerf_fwd(_coords(0), P)
    assert out.shape == (0, 4)
    c = _coords(700, seed=3)
    full, _ = ops.nerf_fwd(c, P)
    out = torch.full((700, 4), 7.0, dtype=torch.float16, device="cuda")
    ops.nerf_fwd(c, P, n_dev=torch.tensor([333], dtype=torch.int32, device="cuda"), out=out)
    assert torch.equal(out[:333], full[:333])
    assert bool((out[333:] == 7.0).all())


def test_density_is_the_forward_alpha_bit_for_bit():
    from jnerf_b200 import ops
    nerf, P = _setup()
    c = _coords(5000, seed=4)
    out, _ = ops.nerf_fwd(c, P)
    sigma = ops.nerf_density(c[:, :3].contiguous(), P)
    assert torch.equal(sigma, out[:, 3])


def test_backward_matches_autograd_and_is_deterministic():
    from jnerf_b200 import ops
    nerf, P = _setup()
    n = 128 * 20 + 77
    c = _coords(n, seed=5)
    g = torch.Generator(device="cuda").manual_seed(6)
    dout = (torch.randn((n, 4), device="cuda", generator=g) * 0.1).half()
    out, saved = ops.nerf_fwd(c, P, save=True)
    grad = ops.nerf_bwd(P, saved, dout)
    grad2 = ops.nerf_bwd(P, saved, dout)
    assert torch.equal(grad, grad2)
    _, saved3 = ops.nerf_fwd(c, P, save=True)
    assert torch.equal(grad, ops.nerf_bwd(P, saved3, dout))
    ref = {k: (W.clone().requires_grad_(), b.clone().requires_grad_()) for k, (W, b) in nerf.unpack(P).items()}
    (_torch_chain(nerf, ref, c) * dout.float()).sum().backward()
    got = nerf.unpack(grad)
    # fp16 activations and fp16 pre-activation gradients (2^-11 each, the kernels' ReLU masks read the fp16 activations) through up to ten
    # layers: 10 % of the gradient's norm per tensor
    rels = {}
    for name, (W, b) in ref.items():
        for k, (tg, tr) in enumerate(((got[name][0], W.grad), (got[name][1], b.grad))):
            rels[name + (".weight", ".bias")[k]] = float((tg - tr).norm() / tr.norm().clamp_min(1e-12))
    print("relative gradient error per tensor:", {k: round(v, 4) for k, v in rels.items()})
    assert max(rels.values()) < 0.1, rels
    # padding of the flat vector receives exactly zero
    pad = nerf_mlp_ref.pad_mask("cuda")
    assert torch.equal(grad[pad], torch.zeros_like(grad[pad]))
    # rows at or past the device row count contribute nothing
    k = 128 * 7 + 5
    gk = ops.nerf_bwd(P, ops.nerf_fwd(c, P, save=True)[1], dout, n_dev=torch.tensor([k], dtype=torch.int32, device="cuda"))
    gs = ops.nerf_bwd(P, ops.nerf_fwd(c[:k].contiguous(), P, save=True)[1], dout[:k].contiguous())
    assert torch.allclose(gk, gs, rtol=1e-5, atol=1e-6)


STEPS = 600
# nerf_base.py's Adam lr of 1e-2 diverges on this stand-in within the first steps, with the kernels and with the fp32 chain alike (the
# loss jumps from 0.3 to 1 and the density grid mean overflows); the usual vanilla-NeRF rate converges
LR = 5e-4


def _train(fp16, steps, seed=5, lr=LR):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, nerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**nerf_cfg(fp16=fp16, synthetic=True, seed=seed, optim=dict(type="Adam", lr=lr, eps=1e-15, betas=(0.9, 0.99))))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 8
    cfg.dataset.train.H = cfg.dataset.train.W = 96
    cfg.dataset.val = None
    r = Runner()
    assert not r.fast
    p0 = r.psnr("train", max_images=2)
    r.train(steps)
    return r, p0, r.psnr("train", max_images=2)


def test_training_fp16_kernels_against_fp32_chain():
    r16, p0, p16 = _train(True, STEPS)
    _, _, p32 = _train(False, STEPS)
    print(f"nerf_cfg lego stand-in, {STEPS} steps: PSNR {p0:.2f} -> fp16 kernels {p16:.2f} dB, fp32 chain {p32:.2f} dB")
    assert p16 > p0 + 3.0, (p0, p16)
    assert abs(p16 - p32) < 1.5, (p16, p32)
    # the whole-frame renderer composites what render_img does (min_transmittance 0), from the same rng position
    s = r16.sampler
    rng0 = s.rng.copy()
    img_ref, _ = r16.render_img_nosync("train", 1)
    s.rng[:] = rng0
    ds = r16.dataset["train"]
    o, d = ds.generate_rays_total_test(1)
    rgb, alpha, _, _ = r16.render_rays(o, d, min_transmittance=0.0)
    img = rgb + torch.tensor(r16.background_color, dtype=torch.float32, device="cuda") * (1 - alpha)
    assert (img.reshape(img_ref.shape) - img_ref).abs().max().item() <= 1e-5
    s.rng[:] = rng0
    img_tiled, _ = r16.render_img("train", 1)
    assert (img_tiled - img_ref).abs().max().item() <= 1e-5
    with pytest.raises(NotImplementedError):
        r16.extract_mesh("/nonexistent-dir-not-created", resolution=8)
