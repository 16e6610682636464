"""The Mip-NeRF sampler kernels (csrc/mip_sampler.cu) at multicam.py's training batch size, against tests/mip_sampler_ref.py:
- mip_sample and mip_resample equal their numpy float32 restatements bit for bit (resample from the kernel's own weights); every
  resampled row is sorted, inside [t_0, t_S] and inside the float64 band of resample_band;
- mip_composite_fwd's weights, rgb, acc and distance lie within composite64's bound, computed from the kernel's own raw and t;
- mip_composite_loss_bwd's rgb and per-ray loss within loss_grad64's bound, every fp32 d(raw) entry within it and every fp16 entry in
  its rn16 bracket (which keeps fp16 subnormals);
- outputs past the last ray keep their NaN sentinel (the C entries are called with oversized NaN-filled buffers), weights_out = NULL
  changes nothing else, and two runs give identical bits.
Cases: one MipRunner.train_step under multicam_cfg (fused fp16, 3072 rays x 128 samples x 2 levels, the multiscale stand-in's lossmult
mask, grad_scale = R) with the reference initialisation and with weights after 300 training steps; one mip_cfg step of the fp32 chain
(1024 rays); S in {1, 2, 3, 4, 5, 31, 32, 33, 127, 128} x R in {1, 7, 8, 9, 257} for fp16 and fp32 raw, white background on and off,
mask None or with zeros; adversarial rows (softplus threshold, saturated colours, T underflowing to 0 or a subnormal, transparent
rays, zero-length intervals, |d| up to 2) and resampling rows whose fp32 CDF dips, all-zero, one-hot and rand^8 rows without padding;
no rays, and the refusal of S = 0 and S = 129 before any launch.  Also the runners' optimizer tail: ngp_adam_ema with fp16 parameters,
fp32 gradients, ema_decay 0 and grad_scale 1 / R against a float64 Adam step by step.

Measured on an H100 80GB HBM3 (700 W power limit); every case prints its own line:
- sample and resample equal the restatements bit for bit on every case, the dipping rows included; no resampled row is out of order.
  In the training steps the resampled fenceposts sit at most 0.86 of the way from the band's centre to its edge; rows with a flat
  stretch reach the edge (u = 0 lands at the end of the stretch, which is the band's end);
- worst error / bound: weights 0.18, rgb 0.15, acc 0.14, distance 0.012, loss 0.13, fp32 d(raw) colour 0.33 and density 0.096; an fp16
  entry's ratio includes half an fp16 ulp and is close to 1 by construction;
- in the multicam step 0.95 M (reference initialisation) and 1.4 M (trained) of the 3.1 M fp16 d(raw) entries are subnormal, and 450
  and 1.3 M are zero; the kernel rounds them correctly;
- Adam: m 0.40, v 0.47, master 0.50 of their bounds; the parameters are rn16(master) and the gradient is left alone;
- the file takes 31 s, the 300 training steps of the trained weights included, with a peak of 7.6 GiB of device memory."""
import time

import numpy as np
import pytest
import torch

import mip_sampler_ref as M
from test_mip_wide_mlp_reference import _weights, step  # noqa: F401  (the module-scoped multicam runner and its trained weights)

pytestmark = pytest.mark.gpu

f32 = np.float32
EXTRA = 3                                       # rays past the last one in every output buffer, NaN-filled


def _np(t):
    return t.detach().cpu().numpy()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape if isinstance(shape, tuple) else (shape,), float("nan"), dtype=dtype, device="cuda")


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------------------------- the C entries
def k_sample(rays, S, lindisp, randomized, rng):
    from jnerf_b200 import lib, ops
    R = rays.shape[0]
    out = _nan((R + EXTRA, S + 1))
    lib.call("ngp_mip_sample", ops._stream(), R, S, ops._p(rays), int(lindisp), int(randomized), int(rng[0]), int(rng[1]), ops._p(out))
    return out


def k_resample(t, w, padding, randomized, rng):
    from jnerf_b200 import lib, ops
    R, S = t.shape[0], t.shape[1] - 1
    out = _nan((R + EXTRA, S + 1))
    lib.call("ngp_mip_resample", ops._stream(), R, S, ops._p(t), ops._p(w), float(padding), int(randomized), int(rng[0]), int(rng[1]), ops._p(out))
    return out


def k_composite(raw, t, rays, p, bias, white, weights=True):
    from jnerf_b200 import lib, ops
    R, S = t.shape[0], t.shape[1] - 1
    rgb, acc, dist = _nan((R + EXTRA, 3)), _nan(R + EXTRA), _nan(R + EXTRA)
    w = _nan((R + EXTRA, S)) if weights else None
    lib.call("ngp_mip_composite_fwd", ops._stream(), R, S, ops._p(raw), ops._dt(raw), ops._p(t), ops._p(rays), float(p), float(bias), int(white),
             ops._p(rgb), ops._p(acc), ops._p(dist), ops._p(w))
    return rgb, acc, dist, w


def k_loss(raw, t, rays, target, mask, p, bias, white, cm, gs):
    from jnerf_b200 import lib, ops
    R, S = rays.shape[0], t.shape[1] - 1
    rgb, loss = _nan((2 * R + EXTRA, 3)), _nan(2 * R + EXTRA)
    draw = _nan((2 * R * S + EXTRA * S, 4), raw.dtype)
    lib.call("ngp_mip_composite_loss_bwd", ops._stream(), R, S, ops._p(raw), ops._dt(raw), ops._p(t), ops._p(rays), ops._p(target), ops._p(mask),
             float(p), float(bias), int(white), float(cm), float(gs), ops._p(rgb), ops._p(loss), ops._p(draw))
    return rgb, loss, draw


def _tails(tally, outs, n_rows, name, tag):
    """Rows [n_rows, ..) of every buffer still NaN; returns the leading rows as numpy."""
    heads = []
    for k, o in enumerate(outs):
        if o is None:
            heads.append(None)
            continue
        n = n_rows[k] if isinstance(n_rows, (list, tuple)) else n_rows
        tally.exact(f"{name} output {k} past the last ray is NaN", _np(torch.isnan(o[n:].float())), tag)
        heads.append(_np(o[:n]))
    return heads


def _same(tally, a, b, name, tag):
    for x, y in zip(a, b):
        if x is not None:
            tally.exact(f"{name}: two runs identical", _np(x.contiguous().view(torch.int8) == y.contiguous().view(torch.int8)), tag)


# ---------------------------------------------------------------------------------------------------------------- checks
def check_sample(tally, rays, S, lindisp, randomized, rng, tag=""):
    a = k_sample(rays, S, lindisp, randomized, rng)
    b = k_sample(rays, S, lindisp, randomized, rng)
    _same(tally, [a], [b], "mip_sample", tag)
    R = rays.shape[0]
    (t,) = _tails(tally, [a], R, "mip_sample", tag)
    want = M.sample_f32(_np(rays), S, lindisp, randomized, rng)
    tally.exact("mip_sample = sample_f32 bit for bit", t.view(np.uint32) == want.view(np.uint32), tag)
    return a[:R]


def check_resample(tally, t, w, padding, randomized, rng, tag="", got=None):
    """got: the kernel's output (as the runner received it), else run here (twice, into NaN-filled buffers)."""
    R = t.shape[0]
    if got is None:
        a = k_resample(t, w, padding, randomized, rng)
        b = k_resample(t, w, padding, randomized, rng)
        _same(tally, [a], [b], "mip_resample", tag)
        (out,) = _tails(tally, [a], R, "mip_resample", tag)
    else:
        out = _np(got)
    tn, wn = _np(t), _np(w)
    want, _ = M.resample_f32(tn, wn, padding, randomized, rng)
    tally.exact("mip_resample = resample_f32 bit for bit", out.view(np.uint32) == want.view(np.uint32), tag)
    tally.exact("resampled rows sorted", np.diff(out, axis=1) >= 0, tag)
    tally.exact("resampled rows inside [t_0, t_S]", (out >= tn[:, :1]) & (out <= tn[:, -1:]), tag)
    for r0 in range(0, R, 512):
        sl = slice(r0, r0 + 512)
        lo, hi = M.resample_band(tn[sl], wn[sl], padding, randomized, _advance(rng, r0 * (t.shape[1])) if randomized else rng)
        r = M.band_ratio(out[sl], lo, hi)
        tally.note("resample position in float64 band", r)
        tally.exact("resample inside the float64 band", r <= 1, tag)


def _advance(rng, n):
    from jnerf_b200 import ops
    return ops.pcg32_advance(np.array(rng, np.uint64).copy(), int(n))


def check_composite(tally, raw, t, rays, p, bias, white, tag="", got=None):
    R = t.shape[0]
    if got is None:
        a = k_composite(raw, t, rays, p, bias, white)
        b = k_composite(raw, t, rays, p, bias, white)
        c = k_composite(raw, t, rays, p, bias, white, weights=False)
        _same(tally, a, b, "mip_composite_fwd", tag)
        _same(tally, a[:3], c[:3], "mip_composite_fwd without weights_out", tag)
        got = _tails(tally, a, R, "mip_composite_fwd", tag)
    else:
        got = [_np(x) if x is not None else None for x in got]
    S = t.shape[1] - 1
    M.check_composite(tally, got, _np(raw).reshape(R, S, 4), _np(t), _np(rays), p, bias, white, tag)


def check_loss(tally, raw, t, rays, target, mask, p, bias, white, cm, gs, tag="", got=None, stats=None):
    R, S = rays.shape[0], t.shape[1] - 1
    if got is None:
        a = k_loss(raw, t, rays, target, mask, p, bias, white, cm, gs)
        b = k_loss(raw, t, rays, target, mask, p, bias, white, cm, gs)
        _same(tally, a, b, "mip_composite_loss_bwd", tag)
        got = _tails(tally, a, [2 * R, 2 * R, 2 * R * S], "mip_composite_loss_bwd", tag)
    else:
        got = [_np(x) for x in got]
    d = M.check_loss(tally, got, _np(raw).reshape(2 * R, S, 4), _np(t), _np(rays), _np(target), None if mask is None else _np(mask), p, bias,
                     white, cm, gs, tag)
    if stats is not None and got[2].dtype == np.float16:
        h = np.abs(got[2].astype(np.float64))
        stats["subnormal"] = stats.get("subnormal", 0) + int(((h > 0) & (h < 2.0 ** -14)).sum())
        stats["zero"] = stats.get("zero", 0) + int((h == 0).sum())
        stats["entries"] = stats.get("entries", 0) + got[2].size


def _finish(name, tally, t0, extra=""):
    print(f"[mip-sampler-fp64] {name}{extra}: worst err/bound {tally.report()}; {time.time() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    assert not tally.fails, tally.fails[:12]


# ---------------------------------------------------------------------------------------------------------------- training steps
def _capture(monkeypatch):
    """Wrap the four sampler entry points of ops; every call's inputs and outputs, cloned, in order."""
    from jnerf_b200 import ops
    calls = []
    cl = lambda x: x.detach().clone() if torch.is_tensor(x) else (np.array(x, copy=True) if isinstance(x, np.ndarray) else x)

    def wrap(name):
        orig = getattr(ops, name)

        def fn(*args, **kw):
            ins = [cl(a) for a in args]
            kws = {k: cl(v) for k, v in kw.items()}
            out = orig(*args, **kw)
            calls.append((name, ins, kws, tuple(cl(o) for o in out) if isinstance(out, tuple) else cl(out)))
            return out
        monkeypatch.setattr(ops, name, fn)
    for name in ("mip_sample", "mip_composite_fwd", "mip_resample", "mip_composite_loss_bwd"):
        wrap(name)
    return calls


def check_step(tally, calls, stats):
    names = [c[0] for c in calls]
    assert names == ["mip_sample", "mip_composite_fwd", "mip_resample", "mip_composite_loss_bwd"], names
    (_, (rays, S, lindisp, randomized, rng), _, t_c) = calls[0]
    want = M.sample_f32(_np(rays), S, lindisp, randomized, rng)
    tally.exact("mip_sample = sample_f32 bit for bit", _np(t_c).view(np.uint32) == want.view(np.uint32), "step: ")
    (_, (raw_c, t, rays_c, p, bias, white, *rest), _, out) = calls[1]
    assert rest in ([], [True])
    check_composite(tally, raw_c, t, rays_c, p, bias, white, "step coarse: ", got=out)
    (_, (t_in, w, padding, randomized_r, rng_r), _, t_f) = calls[2]
    assert torch.equal(w, out[3]) and torch.equal(t_in, t_c)
    check_resample(tally, t_in, w, padding, randomized_r, rng_r, "step resample: ", got=t_f)
    (_, args, kw, out) = calls[3]
    raw, t2, rays2, target, mask, p2, bias2, white2, cm = args[:9]
    gs = kw.get("grad_scale", args[9] if len(args) > 9 else 1.0)
    assert torch.equal(t2, torch.cat([t_c, t_f]))
    check_loss(tally, raw, t2, rays2, target, mask, p2, bias2, white2, cm, gs, "step loss: ", got=out, stats=stats)
    return dict(R=rays.shape[0], S=S, padding=padding, cm=cm, gs=gs, mask=None if mask is None else sorted(set(_np(mask).tolist())),
                dtype=str(raw.dtype).replace("torch.", ""))


@pytest.mark.parametrize("kind", ["init", "trained"])
def test_multicam_step(step, kind, monkeypatch):  # noqa: F811
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    r, trained = step
    r.model.params.data.copy_(trained if kind == "trained" else _weights("init"))
    calls = _capture(monkeypatch)
    r.train_step()
    torch.cuda.synchronize()
    monkeypatch.undo()
    tally, stats = M.Tally(), {}
    info = check_step(tally, calls, stats)
    assert info["R"] == 3072 and info["S"] == 128 and info["dtype"] == "float16" and info["gs"] == 3072.0 and info["cm"] == 0.1
    assert info["padding"] == pytest.approx(0.01) and info["mask"] is not None and len(info["mask"]) > 1
    _finish(f"multicam step/{kind}", tally, t0, f" ({info}; fp16 d(raw): {stats['subnormal']} of {stats['entries']} entries subnormal,"
                                                f" {stats['zero']} zero)")


def test_mip_fp32_step(tmp_path, monkeypatch):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.mip_runner import MipRunner, mip_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    get_cfg().clear()
    update_cfg(**mip_cfg(using_fp16=False, seed=5, log_dir=str(tmp_path)))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=20, H=64, W=64, batch_size=1024 if split == "train" else 64)
    r = MipRunner()
    calls = _capture(monkeypatch)
    r.train_step()
    torch.cuda.synchronize()
    monkeypatch.undo()
    tally = M.Tally()
    info = check_step(tally, calls, {})
    assert info["R"] == 1024 and info["dtype"] == "float32" and info["gs"] == 1.0 and info["mask"] is None
    _finish("mip_cfg fp32 step", tally, t0, f" ({info})")


# ---------------------------------------------------------------------------------------------------------------- edge batches
P, BIAS, CM = 0.001, -1.0, 0.1


def _batch_checks(tally, b, dtypes, tag, stats=None):
    R = b["rays"].shape[0]
    rays = _cu(b["rays"])
    t = _cu(b["t"])
    for dt in dtypes:
        raw = _cu(b["raw"].reshape(-1, 4)).to(dt)
        S = b["raw"].shape[1]
        for white in (False, True):
            for mask in b["masks"]:
                tg = f"{tag}/{str(dt)[6:]}/white={int(white)}/mask={'none' if mask is None else 'zeros'}: "
                check_composite(tally, raw[:R * S], t[:R], rays, P, BIAS, white, tg)
                check_loss(tally, raw, t, rays, _cu(b["target"]), None if mask is None else _cu(mask), P, BIAS, white, CM, float(R), tg, stats=stats)


@pytest.mark.parametrize("S", M.EDGE_S)
def test_edge_batches(S):
    from jnerf_b200 import ops
    t0 = time.time()
    tally = M.Tally()
    for R in M.EDGE_R:
        b = M.edge_batch(R, S, seed=1000 * R + S)
        rays = _cu(b["rays"])
        for lindisp in (False, True):
            for randomized in (False, True):
                check_sample(tally, rays, S, lindisp, randomized, M.pcg_state(R + S), f"R{R}/S{S}: ")
        _batch_checks(tally, b, (torch.float16, torch.float32), f"R{R}/S{S}")
        t = _cu(b["t"][:R])
        w = ops.mip_composite_fwd(_cu(b["raw"][:R].reshape(-1, 4)).half(), t, rays, P, BIAS, False)[3]
        for padding in (0.01, 0.0):
            for randomized in (False, True):
                check_resample(tally, t, w, padding, randomized, M.pcg_state(7 * R + S), f"R{R}/S{S}/pad={padding}: ")
    _finish(f"edge S={S}", tally, t0)


@pytest.mark.parametrize("case", ["fp16-S128", "fp32-S128", "fp16-S33"])
def test_adversarial_rows(case):
    t0 = time.time()
    tally = M.Tally()
    S = int(case.split("-S")[1])
    fp16 = case.startswith("fp16")
    b = M.adversarial_batch(seed=910 + S + fp16, S=S, fp16=fp16)
    _batch_checks(tally, b, (torch.float16,) if fp16 else (torch.float32,), case)
    _finish(f"adversarial {case}", tally, t0)


@pytest.mark.parametrize("S", [4, 33, 127, 128])
def test_resampling_hard_rows(S):
    """Rows whose fp32 CDF dips, all-zero, one-hot and rand^8 rows; padding 0 (and the configs' 0.01)."""
    t0 = time.time()
    tally = M.Tally()
    for padding in (0.0, 0.01):
        w, kinds = M.resample_rows(S, seed=S, padding=padding)
        if padding == 0.0 and S >= 33:
            assert kinds.count("dip") == 8, kinds
        R = w.shape[0]
        t = _cu(M.sample_f32(M.rays_np(R, seed=S), S, False, True, M.pcg_state(S)))
        for randomized in (False, True):
            check_resample(tally, t, _cu(w), padding, randomized, M.pcg_state(S + 3), f"S{S}/pad={padding}: ")
    _finish(f"resampling rows S={S}", tally, t0)


def test_no_rays_and_refused_sample_counts():
    """R = 0 writes nothing; S = 0 (every entry) and S = 129 (those with per-warp shared memory: resample, composite, loss) are refused
    before any launch, leaving the outputs as they were."""
    from jnerf_b200 import lib, ops
    rays = _cu(M.rays_np(4, seed=1))
    rng = M.pcg_state(1)
    t = k_sample(rays, 128, False, True, rng)[:4].contiguous()
    w = torch.rand((4, 128), device="cuda")
    raw = torch.zeros((8 * 128, 4), dtype=torch.float16, device="cuda")
    target = torch.rand((4, 3), device="cuda")
    for S, refused in ((None, False), (0, True), (129, True)):
        n = 0 if S is None else 4
        S_ = 128 if S is None else S
        out = _nan((4, 130))
        o3, o1, o1b = _nan((8, 3)), _nan(8), _nan(8)
        d16 = _nan((8 * 130, 4), torch.float16)
        calls = [("ngp_mip_resample", (n, S_, ops._p(t), ops._p(w), 0.01, 1, int(rng[0]), int(rng[1]), ops._p(out))),
                 ("ngp_mip_composite_fwd", (n, S_, ops._p(raw), ops._dt(raw), ops._p(t), ops._p(rays), 0.001, -1.0, 0, ops._p(o3), ops._p(o1), ops._p(o1b),
                                            ops._p(out))),
                 ("ngp_mip_composite_loss_bwd", (n, S_, ops._p(raw), ops._dt(raw), ops._p(t), ops._p(rays), ops._p(target), None, 0.001, -1.0, 0, 0.1, 1.0,
                                                 ops._p(o3), ops._p(o1), ops._p(d16)))]
        if S != 129:
            calls.append(("ngp_mip_sample", (n, S_, ops._p(rays), 0, 1, int(rng[0]), int(rng[1]), ops._p(out))))
        for name, args in calls:
            if refused:
                with pytest.raises(lib.NgpError, match="n_samples"):
                    lib.call(name, ops._stream(), *args)
            else:
                lib.call(name, ops._stream(), *args)
        torch.cuda.synchronize()
        for buf in (out, o3, o1, o1b, d16):
            assert bool(torch.isnan(buf.float()).all()), (S, name)
    assert ops.mip_sample(rays[:0], 128, False, True, rng).shape == (0, 129)


# ---------------------------------------------------------------------------------------------------------------- optimizer tail
def _adam64(g, m, v, master, lr, step, b1, b2, eps, gs):
    """One jt.nn.Adam step in float64 from the kernel's own state, with the kernel's fp32 hyper-parameters; ema_decay 0 keeps p."""
    b1, b2, eps, lr, gs = (float(f32(x)) for x in (b1, b2, eps, lr, gs))
    ss = lr * np.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    g = g * gs
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    em = 3 * M.U * (b1 * np.abs(m) + (1 - b1) * np.abs(g)) + M.TINY
    ev = 4 * M.U * (b2 * v + (1 - b2) * g * g) + M.TINY
    den = np.sqrt(v1) + eps
    upd = m1 * ss / den
    p = master - upd
    # the update from the kernel's own m1: step size (u), product, sqrt, + eps, quotient; m1's and v1's errors carried
    ep = M.U * np.abs(p) + np.abs(upd) * 6 * M.U + ss / den * em + np.abs(upd) / den * ev / (2 * np.sqrt(v1) + 1e-300) + M.TINY
    return m1, em, v1, ev, p, ep


@pytest.mark.parametrize("degs", [8, 16, "tail"])
def test_adam_step_of_the_mip_runners(degs):
    """ngp_adam_ema as MipRunner / PixelNeRFRunner call it: fp16 parameters, fp32 gradients, ema_decay 0, grad_scale 1 / R, no zeroing;
    at the Mip parameter counts and at counts with n % 4 = 1, 2, 3 (the scalar tail).  Five steps, each against a float64 Adam started
    from the kernel's own m, v and master: m, v and master within a few u, param == rn16(master), the gradient untouched."""
    from jnerf_b200 import ops
    counts = [ops.mip_param_count(degs)] if degs != "tail" else [1, 2, 3, 4097, 1030, 12347]
    R = 3072
    lr, b1, b2, eps = 5e-4, 0.9, 0.99, 1e-15
    tally = M.Tally()
    for n in counts:
        g = torch.Generator(device="cuda").manual_seed(n)
        master = (torch.randn(n, device="cuda", generator=g) * 0.1).half().float()
        param = master.half()
        m = torch.zeros(n, device="cuda")
        v = torch.zeros(n, device="cuda")
        for k in range(1, 6):
            grad = torch.randn(n, device="cuda", generator=g) * R * 10.0 ** torch.empty(n, device="cuda").uniform_(-6, 1, generator=g)
            grad[::7] = 0
            g0, m0, v0, s0 = (_np(x).astype(np.float64) for x in (grad, m, v, master))
            gcopy = grad.clone()
            ops.adam_ema(param, grad, m, v, master, lr, k, b1, b2, eps, 0.0, grad_scale=1.0 / R, zero_grad=False)
            torch.cuda.synchronize()
            m1, em, v1, ev, p, ep = _adam64(g0, m0, v0, s0, lr, k, b1, b2, eps, 1.0 / R)
            tag = f"n={n} step {k}: "
            tally.bound("adam m", _np(m), m1, em, tag)
            tally.bound("adam v", _np(v), v1, ev, tag)
            tally.bound("adam master", _np(master), p, ep, tag)
            tally.exact("param = rn16(master)", _np(param).view(np.uint16) == _np(master).astype(np.float16).view(np.uint16), tag)
            tally.exact("gradient untouched (zero_grad=False)", _np(grad).view(np.uint32) == _np(gcopy).view(np.uint32), tag)
    print(f"[mip-sampler-fp64] adam {degs} (n = {counts}): worst err/bound {tally.report()}")
    assert not tally.fails, tally.fails[:12]
