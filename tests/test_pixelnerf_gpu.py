"""pixelNeRF on the H100 (csrc/pixelnerf.cu) at the training size, 2048 rays x 64 samples x 3 reference views, on the fixture's cameras:
the gather against float64 grid_sample, every forward layer from the saved blocks and every weight and bias gradient against float64
with per-entry bounds, the composite and loss against float64, inference = training bit for bit, seeded determinism, and training
parity with the fp32 torch restatement of Network.py."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "pixelnerf_tiny.npz")
R, S = 2048, 64


def _a(off):
    return (off + 255) // 256 * 256


def saved_offsets(Ms, n_ref):
    """The byte offsets of FwdLayout (csrc/pixelnerf.cu) in training mode."""
    big, small, o, out = Ms * n_ref * 1024, Ms * 1024, 0, {}

    def take(name, b):
        nonlocal o
        out[name] = o
        o += _a(b)
    take("enc", Ms * 128)
    take("taps", Ms * n_ref * 16)
    take("tapw", Ms * n_ref * 16)
    take("s", small)
    take("tmp", big)
    take("mean", small)
    take("x0", big)
    take("h0", big)
    for i in range(3):
        if i:
            take(f"x{i}", big)
            take(f"h{i}", big)
        take(f"g{i}", big)
        take(f"r{i}", big)
    for i in range(2):
        take(f"f2h{i}", small)
        take(f"f2r{i}", small)
        take(f"f2out{i}", small)
    return out


@pytest.fixture(scope="module")
def setup():
    from jnerf_b200.plugin import pixelnerf as pn
    data = pn.TinyNerfData(FIXTURE, 3)
    enc = pn.ImageEncoder(seed=0)
    ref = pn.ReferenceViews(data.images[:3], data.poses[:3], data.focal, enc)
    g = torch.Generator(device="cuda").manual_seed(0)
    rays = next(iter(data.batches(R, g)))
    z = 2.0 + 4.0 * (torch.linspace(0, 1, S + 1, device="cuda")[:-1] + torch.rand(S, generator=g, device="cuda") / S)
    return pn, data, ref, rays[:, :6].contiguous(), rays[:, 6:9].contiguous(), z


def _view(buf, off, rows, cols):
    return buf[off:off + rows * cols * 2].view(torch.float16).view(rows, cols)


U = 2.0 ** -11          # fp16 unit roundoff
SUB = 2.0 ** -25        # half the fp16 subnormal spacing


def _pts64(rays, z):
    return (rays[:, None, :3].double() + rays[:, None, 3:6].double() * z[None, :, None].double()).reshape(-1, 3)


def _fail(name, got, want, bound):
    ok = (got - want).abs() <= bound
    if not ok.all():
        i = tuple(torch.nonzero(~ok)[0].tolist())
        pytest.fail(f"{name} entry {i}: got {got[i].item()} want {want[i].item()} bound {bound[i].item()}; {(~ok).sum().item()} entries out of bound")


@pytest.mark.parametrize("pixel_aligned", [False, True])
def test_gather_matches_float64_grid_sample(setup, pixel_aligned):
    """With W_img = I and b = 0 in f1.0, the saved g_0 = relu(features) = the gathered features (the encoder's maps are >= 0).  Bound: fp16
    rounding of the result + the largest neighbouring-texel step times a few fp32 ulps of uv times (fw - 1) / 2.  Points that clamp to a
    corner of reference 0 (just in front of / behind its image plane, far off axis) and points at its centre (uv = 0 / 0) are held to
    the corner texel exactly, without the ulp term."""
    from jnerf_b200 import ops
    pn, data, ref, rays, _, z = setup
    rays = rays.clone()
    c2w = torch.from_numpy(data.poses[0]).cuda()
    Rm, c = c2w[:3, :3], c2w[:3, 3]
    rays[8:16, 3:6] = Rm[:, 2]                                            # behind reference 0 (its +z axis)
    rays[16:24, 3:6] *= torch.tensor([40.0, -40.0, 1.0], device="cuda")   # far off every frustum
    side = torch.tensor([1.0, 1.0, 1.0, 1.0, -1.0, -1.0, -1.0, -1.0], device="cuda")
    rays[24:32, :3] = c + Rm[:, 0] + 0.5 * Rm[:, 1] + 1e-3 * side[:, None] * Rm[:, 2]   # p = (1, 0.5, +-1e-3): |uv| ~ 10^3
    rays[24:32, 3:6] = 1e-7 * Rm[:, 0]
    rays[32:36, :3] = c                                                   # the camera centre: p = 0, uv = NaN
    rays[32:36, 3:6] = 0.0
    state = pn.init_state(1)
    state["f1.0.img_mlp.0.weight"] = torch.eye(512)
    state["f1.0.img_mlp.0.bias"] = torch.zeros(512)
    m = pn.PixelNeRF(state)
    Ms = R * S
    saved = torch.empty(ops.pixelnerf_workspace_bytes(Ms, 3)[0], dtype=torch.uint8, device="cuda")
    ops.pixelnerf_fwd(rays, z, m.params, ref.feats, ref.cams, ref.scale, pixel_aligned, saved=saved)
    torch.cuda.synchronize()
    got = _view(saved, saved_offsets(Ms, 3)["g0"], 3 * Ms, 512).double().view(3, Ms, 512)
    assert torch.isfinite(got).all()
    pts = _pts64(rays, z)
    uv = pn.project(pts, ref.cams.double(), ref.scale, pixel_aligned)
    uv = torch.nan_to_num(uv, nan=-1.0)                  # torch's CUDA grid_sample: a NaN coordinate clamps to the first texel
    f = ref.feats.double().permute(0, 3, 1, 2)
    want = torch.nn.functional.grid_sample(f, uv[:, :, None, :], align_corners=True, padding_mode="border")[..., 0].permute(0, 2, 1)
    fh, fw = ref.feats.shape[1:3]
    step = max((ref.feats[:, 1:] - ref.feats[:, :-1]).abs().max().item(), (ref.feats[:, :, 1:] - ref.feats[:, :, :-1]).abs().max().item())
    ulp = uv.abs().clamp_min(1.0) * 2.0 ** -23
    bound = want.abs() * U + 2.0 ** -24 + step * 8 * ulp.max(-1).values[..., None] * (max(fh, fw) - 1) / 2
    _fail("gather", got, want, bound)
    # the clamped and the 0 / 0 points of reference 0: a corner texel, exactly
    corner = (uv[0].abs() > 100).all(-1)
    assert corner[24 * S:32 * S].all()
    fr = ref.feats[0].double()
    sgn = torch.sign(uv[0, 24 * S:32 * S])
    iy = ((sgn[:, 1] + 1) / 2 * (fh - 1)).long()
    ix = ((sgn[:, 0] + 1) / 2 * (fw - 1)).long()
    assert torch.equal(got[0, 24 * S:32 * S], fr[iy, ix])
    assert torch.equal(got[0, 32 * S:36 * S], fr[0, 0].expand(4 * S, -1))
    nan_grid = torch.full((1, 4, 1, 2), float("nan"), device="cuda")
    assert torch.equal(torch.nn.functional.grid_sample(ref.feats[:1].float().permute(0, 3, 1, 2), nan_grid, align_corners=True,
                                                       padding_mode="border")[0, :, 0, 0].double(), fr[0, 0])


def _lin_check(name, X, W, b, got, relu=True):
    """One Linear from its fp16 inputs as the kernel read them: y = act(X W^T + b) in float64.  Bound: the fp16 rounding of y plus
    fp32 accumulation over K terms, (K + 2) 2^-24 (|X| |W|^T + |b|)."""
    acc = X @ W.t() + b
    want = torch.relu(acc) if relu else acc
    mag = X.abs() @ W.abs().t() + b.abs()
    _fail(name, got, want, U * want.abs() + SUB + (X.shape[1] + 2) * 2.0 ** -24 * mag)


def test_forward_layer_by_layer_and_inference_is_bit_identical(setup):
    """Every layer of the training forward at 2048 x 64 x 3, from the saved fp16 blocks, against float64 with per-entry bounds."""
    from jnerf_b200 import ops
    pn, data, ref, rays, _, z = setup
    m = pn.PixelNeRF(seed=3)
    Ms = R * S
    saved = torch.empty(ops.pixelnerf_workspace_bytes(Ms, 3)[0], dtype=torch.uint8, device="cuda")
    raw = ops.pixelnerf_fwd(rays, z, m.params, ref.feats, ref.cams, ref.scale, saved=saved)
    raw_inf = ops.pixelnerf_fwd(rays, z, m.params, ref.feats, ref.cams, ref.scale)
    torch.cuda.synchronize()
    assert torch.equal(raw.view(torch.int16), raw_inf.view(torch.int16))
    assert torch.isfinite(raw).all()
    st = {k: v.cuda().half().double() for k, v in m.reference_state().items()}
    off = saved_offsets(Ms, 3)
    V = lambda name, rows, cols=512: _view(saved, off[name], rows, cols).double()
    # the encoding: fp32 x = o + d z, 2^i 1.5 x, sin / cos, each within a few fp32 ulps, then rounded to fp16
    pts = _pts64(rays, z)
    want = pn.positional_encoding(pts, rays[:, None, 3:6].double().expand(-1, S, -1).reshape(-1, 3))
    enc = V("enc", Ms, 64)
    assert torch.all(enc[:, 42:] == 0)
    xa = (rays[:, None, :3].double().abs() + rays[:, None, 3:6].double().abs() * z[None, :, None].double().abs()).reshape(-1, 3)
    arg = torch.cat([xa * 2.0 ** -22] + [xa * 2.0 ** i * 1.5 * 2.0 ** -21 + 2.0 ** -21 for i in range(6) for _ in (0, 1)] + [xa * 0 + 2.0 ** -21], -1)
    _fail("enc", enc[:, :42], want, U * want.abs() + SUB + arg)
    feat = pn.feature_matching(ref.feats.double(), pts, ref.cams.double(), ref.scale)       # (3, Ms, 512); the gather is checked above
    uv = torch.nan_to_num(pn.project(pts, ref.cams.double(), ref.scale), nan=-1.0)
    step = max((ref.feats[:, 1:] - ref.feats[:, :-1]).abs().max().item(), (ref.feats[:, :, 1:] - ref.feats[:, :, :-1]).abs().max().item())
    tap = (step * 8 * uv.abs().clamp_min(1.0).amax(-1) * 2.0 ** -23 * (max(ref.feats.shape[1:3]) - 1) / 2)[..., None]   # (3, Ms, 1)
    s = V("s", Ms)
    _lin_check("mlp.0", enc[:, :42], st["mlp.0.weight"], st["mlp.0.bias"], s)
    res = s[None].expand(3, -1, -1)
    for i in range(3):
        W, b = st[f"f1.{i}.img_mlp.0.weight"], st[f"f1.{i}.img_mlp.0.bias"]
        g = V(f"g{i}", 3 * Ms).view(3, Ms, 512)
        acc = feat @ W.t() + b
        mag = feat.abs() @ W.abs().t() + b.abs()
        want = torch.relu(acc)
        # the features enter as fp16: U |F| |W| more
        _fail(f"f1.{i}.img_mlp.0", g, want, U * want.abs() + SUB + (U + 514 * 2.0 ** -24) * mag + tap * W.abs().sum(1))
        x = V(f"x{i}", 3 * Ms).view(3, Ms, 512)
        want = res + g
        _fail(f"f1.{i} x", x, want, U * want.abs() + SUB)
        h = V(f"h{i}", 3 * Ms)
        _lin_check(f"f1.{i}.mlp.0", x.reshape(-1, 512), st[f"f1.{i}.mlp.0.weight"], st[f"f1.{i}.mlp.0.bias"], h)
        r = V(f"r{i}", 3 * Ms)
        _lin_check(f"f1.{i}.mlp.2", h, st[f"f1.{i}.mlp.2.weight"], st[f"f1.{i}.mlp.2.bias"], r)
        res = (r.view(3, Ms, 512) + x).half().double()                   # the block output, rounded once to fp16
    mean = V("mean", Ms)
    want = res.sum(0) / 3
    _fail("mean", mean, want, U * want.abs() + SUB + 3 * 2.0 ** -24 * res.abs().sum(0))
    x = mean
    for i in range(2):
        h = V(f"f2h{i}", Ms)
        _lin_check(f"f2.{i}.mlp.0", x, st[f"f2.{i}.mlp.0.weight"], st[f"f2.{i}.mlp.0.bias"], h)
        r = V(f"f2r{i}", Ms)
        _lin_check(f"f2.{i}.mlp.2", h, st[f"f2.{i}.mlp.2.weight"], st[f"f2.{i}.mlp.2.bias"], r)
        out = V(f"f2out{i}", Ms)
        want = r + x
        _fail(f"f2.{i} out", out, want, U * want.abs() + SUB)
        x = out
    acc = x @ st["final_layer.weight"].t() + st["final_layer.bias"]
    mag = x.abs() @ st["final_layer.weight"].abs().t() + st["final_layer.bias"].abs()
    want = torch.cat([torch.relu(acc[:, :1]), torch.sigmoid(acc[:, 1:])], -1)
    slope = torch.tensor([1.0, 0.25, 0.25, 0.25], dtype=torch.float64, device="cuda")
    _fail("final_layer", raw.double(), want, U * want.abs() + SUB + slope * 514 * 2.0 ** -24 * mag + 2.0 ** -22)


def test_backward_matches_float64_at_training_size(setup):
    """The backward at 2048 x 64 x 3 against a float64 backward that reads the same saved fp16 activations and ReLU masks (so no mask
    differs), from the same d(raw).  Per entry: |got - want| <= 2 (sum_m E|X| + 2^-11 sum |dY||X|), where E bounds the error the kernel's
    dY carries: its own fp16 rounding (2^-11 |dY|, and 2^-25 below the normal range), fp32 accumulation, and the error of the gradients it
    was formed from, carried through |W| layer by layer.  Per tensor: ||got - want|| <= 1e-2 ||want|| (measured: at most 6.7e-4), which a
    gradient 10 % too small or too large, a lost wgrad chunk or a lost reference fails."""
    from jnerf_b200 import ops
    pn, data, ref, rays, _, z = setup
    m = pn.PixelNeRF(seed=4)
    Ms = R * S
    saved = torch.empty(ops.pixelnerf_workspace_bytes(Ms, 3)[0], dtype=torch.uint8, device="cuda")
    raw = ops.pixelnerf_fwd(rays, z, m.params, ref.feats, ref.cams, ref.scale, saved=saved)
    g = torch.Generator(device="cuda").manual_seed(5)
    draw = (torch.randn((Ms, 4), generator=g, device="cuda") * 0.5).half()
    grad = ops.pixelnerf_bwd(R, S, m.params, ref.feats, saved, raw, draw)
    grad2 = ops.pixelnerf_bwd(R, S, m.params, ref.feats, saved, raw, draw)
    torch.cuda.synchronize()
    assert torch.equal(grad, grad2)
    got = pn.unpack(grad)
    st = {k: v.cuda().half().double() for k, v in m.reference_state().items()}
    off = saved_offsets(Ms, 3)
    V = lambda name, rows, cols=512: _view(saved, off[name], rows, cols).double()
    want, bound = {}, {}
    rnd = lambda v: U * v.abs() + SUB                                  # the fp16 rounding of one stored gradient

    def wgrad(name, dy, e, x, x_rounded=False):
        want[f"{name}.weight"] = dy.t() @ x
        want[f"{name}.bias"] = dy.sum(0)
        mag = dy.abs().t() @ x.abs()
        bound[f"{name}.weight"] = e.t() @ x.abs() + (2 * U if x_rounded else U) * mag
        bound[f"{name}.bias"] = e.sum(0) + U * dy.abs().sum(0)

    def dgrad(dy, e, W):
        """dy W and the error of the kernel's result before its own rounding: the carried error through |W| + fp32 accumulation."""
        return dy @ W, e @ W.abs() + (W.shape[0] + 2) * 2.0 ** -24 * (dy.abs() @ W.abs())
    rw, dw = raw.double(), draw.double()
    dpre = torch.stack([dw[:, 0] * (rw[:, 0] > 0), *[dw[:, c] * rw[:, c] * (1 - rw[:, c]) for c in (1, 2, 3)]], 1)
    e_pre = rnd(dpre) + 2.0 ** -22 * dw.abs()
    wgrad("final_layer", dpre, e_pre, V("f2out1", Ms))
    d, e = dgrad(dpre, e_pre, st["final_layer.weight"])
    e = e + rnd(d)
    for i in (1, 0):
        xin = V("mean", Ms) if i == 0 else V(f"f2out{i - 1}", Ms)
        h, r = V(f"f2h{i}", Ms), V(f"f2r{i}", Ms)
        dr, e_dr = d * (r > 0), e * (r > 0)
        wgrad(f"f2.{i}.mlp.2", dr, e_dr, h)
        dh, e_dh = dgrad(dr, e_dr, st[f"f2.{i}.mlp.2.weight"])
        dh, e_dh = dh * (h > 0), (e_dh + rnd(dh)) * (h > 0)
        wgrad(f"f2.{i}.mlp.0", dh, e_dh, xin)
        dx, e_dx = dgrad(dh, e_dh, st[f"f2.{i}.mlp.0.weight"])
        d = dx + d
        e = e_dx + e + rnd(d)
    # the mean's gradient, split over the references (the kernel rounds d / 3 once more for the ReLU-masked copy)
    d = (d / 3)[None].expand(3, -1, -1).reshape(-1, 512)
    e = (e / 3 + rnd(d[:Ms]))[None].expand(3, -1, -1).reshape(-1, 512)
    feat = pn.feature_matching(ref.feats.double(), _pts64(rays, z), ref.cams.double(), ref.scale).reshape(-1, 512)
    for i in (2, 1, 0):
        x, h, r, gg = V(f"x{i}", 3 * Ms), V(f"h{i}", 3 * Ms), V(f"r{i}", 3 * Ms), V(f"g{i}", 3 * Ms)
        dr, e_dr = d * (r > 0), e * (r > 0)
        wgrad(f"f1.{i}.mlp.2", dr, e_dr, h)
        dh, e_dh = dgrad(dr, e_dr, st[f"f1.{i}.mlp.2.weight"])
        dh, e_dh = dh * (h > 0), (e_dh + rnd(dh)) * (h > 0)
        del dr, e_dr, h, r
        wgrad(f"f1.{i}.mlp.0", dh, e_dh, x)
        dx, e_dx = dgrad(dh, e_dh, st[f"f1.{i}.mlp.0.weight"])
        d = dx + d
        e = e_dx + e + rnd(d)
        del dx, e_dx, dh, e_dh, x
        wgrad(f"f1.{i}.img_mlp.0", d * (gg > 0), e * (gg > 0), feat, x_rounded=True)
        del gg
    sm = V("s", Ms) > 0
    ds = d.view(3, Ms, 512).sum(0)
    e_ds = (e.view(3, Ms, 512).sum(0) + 3 * 2.0 ** -24 * d.view(3, Ms, 512).abs().sum(0) + rnd(ds)) * sm
    wgrad("mlp.0", ds * sm, e_ds, V("enc", Ms, 64)[:, :42])
    worst_entry, worst_norm = {}, {}
    for k, w in want.items():
        err = (got[k].double() - w).abs()
        worst_entry[k] = (err / (bound[k] + 1e-30)).max().item()
        worst_norm[k] = ((got[k].double() - w).norm() / w.norm()).item()
    print("worst |error| / bound:", {k: round(v, 3) for k, v in worst_entry.items()})
    print("||error|| / ||gradient||:", {k: round(v, 5) for k, v in worst_norm.items()})
    assert max(worst_entry.values()) <= 2, {k: v for k, v in worst_entry.items() if v > 2}
    assert max(worst_norm.values()) <= 1e-2, {k: v for k, v in worst_norm.items() if v > 1e-2}


def test_composite_and_loss_match_float64(setup):
    from jnerf_b200 import ops
    pn, data, ref, rays, target, z = setup
    g = torch.Generator(device="cuda").manual_seed(6)
    raw = torch.rand((R * S, 4), generator=g, device="cuda")
    raw[:, 0] = torch.relu(raw[:, 0] * 4 - 1)
    raw = raw.half()
    rgb, depth, acc = ops.pixelnerf_composite_fwd(raw, z, rays)
    rgb2, loss, draw = ops.pixelnerf_composite_loss_bwd(raw, z, rays, target, grad_scale=float(R))
    r64 = raw.double().requires_grad_()
    w_rgb, w_depth, w_acc = pn.composite_torch(r64, z.double(), rays.double())
    mse = ((w_rgb - target.double()) ** 2).mean()
    (mse * R).backward()
    assert (rgb.double() - w_rgb).abs().max() < 1e-5 and torch.equal(rgb, rgb2)
    assert (depth.double() - w_depth).abs().max() < 1e-4 and (acc.double() - w_acc).abs().max() < 1e-5
    assert abs(loss.sum().item() - mse.item()) < 1e-6 * max(1.0, mse.item())
    gw = r64.grad.clamp(-65504, 65504)
    err = (draw.double() - gw).abs()
    assert (err <= gw.abs() * 2e-3 + 1e-6).all(), err.max()


def test_two_seeded_runs_are_bit_identical(setup):
    from jnerf_b200.pixelnerf_runner import PixelNeRFRunner, pixelnerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    runs = []
    for _ in range(2):
        get_cfg().clear()
        update_cfg(**pixelnerf_cfg(FIXTURE, seed=7))
        r = PixelNeRFRunner()
        r.train(steps=20)
        torch.cuda.synchronize()
        runs.append(r.model.master.clone())
    assert torch.equal(runs[0], runs[1])


# Training parity, measured on an H100 80GB HBM3 with the seeded He-initialised encoder, 112 steps (8 epochs) from the same weights, batches
# and depths: fused 9.575 -> 12.043 dB, fp32 torch 9.576 -> 12.086 dB (rises 2.47 and 2.51 dB, 0.043 dB apart).  The floor is half the
# smaller rise; the tolerance about five times the measured gap.
PARITY_STEPS = 112
PARITY_MIN_RISE_DB = 1.2
PARITY_TOL_DB = 0.2


def _torch_psnr(pn, runner, state):
    """Held-out PSNR of the fp32 torch chain at the runner's mid-interval depths."""
    z = runner._z(randomized=False)
    ref, data = runner.ref, runner.data
    feats = ref.feats.float()
    out = []
    with torch.no_grad():
        for i in range(data.n_train, data.images.shape[0]):
            rays = data.image_rays(data.poses[i])
            rgb = []
            for p in range(0, rays.shape[0], 1024):
                r = rays[p:p + 1024]
                pts = (r[:, None, :3] + r[:, None, 3:6] * z[None, :, None]).reshape(-1, 3)
                enc = pn.positional_encoding(pts, r[:, None, 3:6].expand(-1, z.shape[0], -1).reshape(-1, 3))
                raw = pn.network_torch(state, enc, pn.feature_matching(feats, pts, ref.cams, ref.scale))
                rgb.append(pn.composite_torch(raw, z, r)[0])
            img = torch.cat(rgb).reshape(data.H, data.W, 3)
            mse = ((img - torch.from_numpy(data.images[i]).cuda()) ** 2).mean()
            out.append(float(-10.0 * torch.log10(mse)))
    return sum(out) / len(out)


def test_training_parity_with_the_fp32_torch_network(setup):
    """The fused path and the fp32 torch restatement (network_torch, composite_torch, torch.optim.Adam with main.py's settings) train from
    the same initial weights on the same batches and depths; both held-out PSNRs rise and end close together."""
    from jnerf_b200.pixelnerf_runner import PixelNeRFRunner, pixelnerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    pn = setup[0]
    get_cfg().clear()
    update_cfg(**pixelnerf_cfg(FIXTURE, seed=11))
    fused = PixelNeRFRunner()
    twin = PixelNeRFRunner()                               # same seed: same weights, batches and depths, drawn in the same order
    state = {k: v.cuda().clone().requires_grad_() for k, v in fused.model.reference_state().items()}
    p0_fused, p0_torch = fused.test(), _torch_psnr(pn, twin, state)
    fused.train(steps=PARITY_STEPS)
    cfg = get_cfg()
    opt = torch.optim.Adam(list(state.values()), lr=cfg.lr, betas=tuple(cfg.betas), eps=cfg.eps)
    done = 0
    feats = twin.ref.feats.float()
    while done < PARITY_STEPS:
        for batch in twin.data.batches(int(cfg.batch_size), twin.gen):
            z = twin._z()
            rays, target = batch[:, :6], batch[:, 6:9]
            pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[None, :, None]).reshape(-1, 3)
            enc = pn.positional_encoding(pts, rays[:, None, 3:6].expand(-1, z.shape[0], -1).reshape(-1, 3))
            raw = pn.network_torch(state, enc, pn.feature_matching(feats, pts, twin.ref.cams, twin.ref.scale))
            loss = ((pn.composite_torch(raw, z, rays)[0] - target) ** 2).mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
            done += 1
            if done == PARITY_STEPS:
                break
    p1_fused, p1_torch = fused.test(), _torch_psnr(pn, twin, state)
    print(f"PARITY fused {p0_fused:.3f} -> {p1_fused:.3f} dB, torch fp32 {p0_torch:.3f} -> {p1_torch:.3f} dB")
    assert p1_fused - p0_fused >= PARITY_MIN_RISE_DB and p1_torch - p0_torch >= PARITY_MIN_RISE_DB
    assert abs(p1_fused - p1_torch) <= PARITY_TOL_DB
