"""Rehearsal of tests/mip_sampler_ref.py on the CPU.

A numpy float32 emulation of ray_forward, mip_composite_fwd_kernel and mip_loss_bwd_kernel (csrc/mip_sampler.cu) in the kernels' order
(lanes of 4 samples, warp_scan, warp_sum, the block's mask sum) is another fp32 evaluation of the same expressions, with expf within
1.5 ulp (a float64 exp rounded to fp32 and moved by a random ulp), so every value it produces must lie within composite64's and
loss_grad64's bounds: the bounds are not too tight.  The same emulation with one expression changed must fail them: the bounds are not
too loose.  The float32 restatements of the sampling kernels stay within the float64 band of mip_cpu_backend on the same uniforms,
with and without resample padding, on rows whose fp32 CDF dips."""
import numpy as np
import pytest
import torch

import mip_cpu_backend as mcb
import mip_sampler_ref as M

f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------- the emulation
def _expf(x, g):
    with np.errstate(over="ignore"):
        y = np.exp(np.asarray(x, np.float64)).astype(f32)
    k = np.where((np.asarray(x) == 0) | (y == 0), 0, g.integers(-1, 2, y.shape))   # expf(0) = 1 and an underflow to 0 are exact
    return np.where(k > 0, np.nextafter(y, f32(np.inf)), np.where(k < 0, np.nextafter(y, f32(0)), y)).astype(f32)


def _log1pf(x):
    return np.log1p(np.asarray(x, np.float64)).astype(f32)


def _lane_sum(x):
    s = np.zeros(x.shape[:2], f32)
    for q in range(4):
        s = (s + x[:, :, q]).astype(f32)
    return s


def ray_forward(raw, t, rays, p, bias, g, mut=()):
    """ray_forward for every ray: dict of (R, 32, 4[, 3]) float32 arrays, sample i = 4 lane + q."""
    R, S = raw.shape[:2]
    d = np.asarray(rays, f32)[:, 3:6]
    dnorm = np.sqrt(((d[:, 0] * d[:, 0]).astype(f32) + (d[:, 1] * d[:, 1]).astype(f32)).astype(f32) + (d[:, 2] * d[:, 2]).astype(f32)).astype(f32)
    if "delta without |d|" in mut:
        dnorm = np.ones_like(dnorm)
    live = M.lanes(np.ones((R, S), bool), False)
    rw = M.lanes(raw.astype(f32))
    k = f32(f32(1) + f32(f32(2) * f32(p)))
    s = (f32(1) / (f32(1) + _expf(-rw[..., :3], g)).astype(f32)).astype(f32)
    c = ((s * k).astype(f32) - f32(p)).astype(f32)
    sg = ((s * (f32(1) - s).astype(f32)).astype(f32) * k).astype(f32)
    x = (rw[..., 3] + f32(bias)).astype(f32)
    sigma = np.where(x > f32(20), x, _log1pf(_expf(x, g)))
    dsig = (f32(1) / (f32(1) + _expf(-x, g)).astype(f32)).astype(f32)
    if "dsig = 1" in mut:
        dsig = np.ones_like(dsig)
    tt = np.asarray(t, f32)
    delta = M.lanes(((tt[:, 1:] - tt[:, :-1]).astype(f32) * dnorm[:, None]).astype(f32))
    sd = np.where(live, (sigma * delta).astype(f32), f32(0))
    c, sg = np.where(live[..., None], c, f32(0)), np.where(live[..., None], sg, f32(0))
    dsig, delta = np.where(live, dsig, f32(0)), np.where(live, delta, f32(0))
    local = _lane_sum(sd)
    before = (M.warp_scan(local) - local).astype(f32)
    tb, w = np.empty_like(sd), np.empty_like(sd)
    for q in range(4):
        tb[..., q] = _expf(-before, g)
        w[..., q] = ((f32(1) - _expf(-sd[..., q], g)).astype(f32) * tb[..., q]).astype(f32)
        before = (before + sd[..., q]).astype(f32)
    return dict(c=c, sg=sg, sd=sd, dsig=dsig, delta=delta, w=w, tb=tb, live=live)


def composite_f32(raw, t, rays, p, bias, white, g, mut=()):
    """mip_composite_fwd_kernel: (rgb (R, 3), acc (R,), distance (R,), weights (R, S))."""
    R, S = raw.shape[:2]
    r = ray_forward(raw, t, rays, p, bias, g, mut)
    w, live = r["w"], r["live"]
    wl = np.where(live, w, f32(0))
    tt = np.asarray(t, f32)
    tm = M.lanes((f32(0.5) * (tt[:, :-1] + tt[:, 1:]).astype(f32)).astype(f32))
    rgb = np.stack([M.warp_sum(_lane_sum((wl * r["c"][..., j]).astype(f32))) for j in range(3)], 1)
    acc = M.warp_sum(_lane_sum(wl))
    wt = M.warp_sum(_lane_sum((wl * tm).astype(f32)))
    if white:
        rgb = (rgb + (f32(1) - acc).astype(f32)[:, None]).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        dist = np.fmin(np.fmax((wt / acc).astype(f32), tt[:, 0]), tt[:, S])
    return rgb, acc, dist, w.reshape(R, -1)[:, :S]


def block_mask_sum(mask, R):
    """The 256-thread block's fp32 mask sum: serial over i = tid, tid + 256, .., then the shared-memory tree."""
    red = np.zeros(256, f32)
    m = np.asarray(mask, f32)
    for i in range(R):
        red[i % 256] = f32(red[i % 256] + m[i])
    h = 128
    while h:
        red[:h] = (red[:h] + red[h:2 * h]).astype(f32)
        h //= 2
    return red[0]


def loss_bwd_f32(raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale, g, dtype, mut=()):
    """mip_loss_bwd_kernel over the 2R rays: (rgb (2R, 3), loss (2R,), draw (2R, S, 4) of dtype)."""
    R = rays.shape[0]
    S = raw.shape[1]
    rays2 = np.concatenate([rays, rays])
    r = ray_forward(raw, t, rays2, p, bias, g, mut)
    msum = f32(R) if (mask is None or "mask sum = R" in mut) else block_mask_sum(mask, R)
    m = np.ones(R, f32) if mask is None else np.asarray(mask, f32)
    m = np.concatenate([m, m])
    mult = np.concatenate([np.full(R, f32(coarse_mult)), np.ones(R, f32)])
    w = r["w"]
    c = np.stack([M.warp_sum(_lane_sum((w * r["c"][..., j]).astype(f32))) for j in range(3)], 1)
    acc = M.warp_sum(_lane_sum(w))
    tg = np.concatenate([target, target]).astype(f32)
    loss = np.zeros(2 * R, f32)
    gr = np.empty((2 * R, 3), f32)
    gs = f32(grad_scale)
    for j in range(3):
        if white:
            c[:, j] = (c[:, j] + (f32(1) - acc).astype(f32)).astype(f32)
        e = (c[:, j] - tg[:, j]).astype(f32)
        loss = (loss + (e * e).astype(f32)).astype(f32)
        gr[:, j] = (gs * ((((mult * f32(2)).astype(f32) * m).astype(f32) * e).astype(f32) / msum).astype(f32)).astype(f32)
        if "grad_scale twice" in mut:
            gr[:, j] = (gr[:, j] * gs).astype(f32)
    lv = ((((mult * m).astype(f32)) * loss).astype(f32) / msum).astype(f32)
    bg = f32(1) if (white and "no white - 1 in gc" not in mut) else f32(0)
    gc = np.zeros(w.shape, f32)
    for j in range(3):
        gc = (gc + (gr[:, None, None, j] * (r["c"][..., j] - bg).astype(f32)).astype(f32)).astype(f32)
    wgc = (w * gc).astype(f32)
    local = _lane_sum(wgc)
    total = M.warp_sum(local)[:, None]
    upto = (M.warp_scan(local) - local).astype(f32)
    out = np.empty((2 * R, 32, 4, 4), f32)
    for q in range(4):
        if "suffix inclusive of i" not in mut:
            upto = (upto + wgc[..., q]).astype(f32)
        tnext = r["tb"][..., q] if "T_i for T_(i+1)" in mut else (r["tb"][..., q] * _expf(-r["sd"][..., q], g)).astype(f32)
        dsd = ((tnext * gc[..., q]).astype(f32) - (total - upto).astype(f32)).astype(f32)
        if "suffix inclusive of i" in mut:
            upto = (upto + wgc[..., q]).astype(f32)
        for j in range(3):
            out[..., q, j] = ((w[..., q] * gr[:, None, j]).astype(f32) * r["sg"][..., q, j]).astype(f32)
        out[..., q, 3] = ((dsd * r["delta"][..., q]).astype(f32) * r["dsig"][..., q]).astype(f32)
    d = out.reshape(2 * R, -1, 4)[:, :S].astype(dtype)
    if "fp16 store flushes subnormals" in mut:
        d = np.where(np.abs(d) < np.float16(2.0 ** -14), np.float16(0), d)
    return c, lv, d


# ---------------------------------------------------------------------------------------------------------------- cases
P, BIAS, CM = 0.001, -1.0, 0.1


def _batches(which):
    if which == "edge":
        return [(f"R{R}/S{S}", M.edge_batch(R, S, seed=1000 * R + S)) for R in M.EDGE_R for S in M.EDGE_S]
    return [(f"adversarial/{name}", M.adversarial_batch(seed=910 + k, S=S, fp16=fp16))
            for k, (name, S, fp16) in enumerate([("fp16-S128", 128, True), ("fp32-S128", 128, False), ("fp16-S33", 33, True)])]


def _run(tally, name, b, dtype, white, mask, g, mut=()):
    raw = b["raw"].astype(dtype)
    R, S = b["rays"].shape[0], raw.shape[1]
    tag = f"{name}/{np.dtype(dtype).name}/white={int(white)}/mask={'none' if mask is None else 'zeros'}: "
    got = composite_f32(raw[:R], b["t"][:R], b["rays"], P, BIAS, white, g, mut)
    M.check_composite(tally, got, raw[:R], b["t"][:R], b["rays"], P, BIAS, white, tag)
    got = loss_bwd_f32(raw, b["t"], b["rays"], b["target"], mask, P, BIAS, white, CM, float(R), g, dtype, mut)
    M.check_loss(tally, got, raw, b["t"], b["rays"], b["target"], mask, P, BIAS, white, CM, float(R), tag)


@pytest.mark.parametrize("which", ["edge", "adversarial"])
def test_kernel_order_emulation_lies_within_the_bounds(which):
    tally = M.Tally()
    g = np.random.default_rng(7)
    for name, b in _batches(which):
        for dtype in (np.float16, np.float32):
            for white in (False, True):
                for mask in b["masks"]:
                    _run(tally, name, b, dtype, white, mask, g)
    print(f"[mip-sampler-bound-cpu] {which}: {tally.report()}")
    assert not tally.fails, tally.fails[:10]
    assert tally.worst["d(raw) density float32"] > 1e-3 and tally.worst["composite w"] > 1e-3, tally.worst


MUTANTS = {
    "T_i for T_(i+1)": "d(raw) density",
    "suffix inclusive of i": "d(raw) density",
    "no white - 1 in gc": "d(raw) density",
    "grad_scale twice": "d(raw) colour",
    "dsig = 1": "d(raw) density",
    "delta without |d|": "composite w",
    "fp16 store flushes subnormals": "d(raw)",
    "mask sum = R": "loss",
}


@pytest.mark.parametrize("mut", list(MUTANTS))
def test_each_mutant_fails_its_bound(mut):
    """One batch of 9 rays of 128 samples, white and black background, masked and not, fp16 and fp32: the mutant fails with the named
    quantity and its first entry."""
    b = M.edge_batch(9, 128, seed=77)
    tally = M.Tally()
    g = np.random.default_rng(8)
    for dtype in (np.float16, np.float32):
        for white in (False, True):
            for mask in b["masks"]:
                _run(tally, "R9/S128", b, dtype, white, mask, g, (mut,))
    hit = [f for f in tally.fails if MUTANTS[mut] in f]
    assert hit, (mut, tally.fails[:4])
    print(f"[mip-sampler-bound-cpu] mutant {mut!r}: {hit[0]}")


# ---------------------------------------------------------------------------------------------------------------- sampling
@pytest.mark.parametrize("lindisp", [False, True])
@pytest.mark.parametrize("randomized", [False, True])
def test_sample_f32_within_float64_band(lindisp, randomized):
    """The fp32 fenceposts within a few fp32 roundings of mip_cpu_backend.sample on the same uniforms (|t| <= 6: 2^-21 absolute)."""
    rays = M.rays_np(33, seed=3)
    for S in M.EDGE_S:
        rng = M.pcg_state(S)
        t = M.sample_f32(rays, S, lindisp, randomized, rng)
        u = torch.from_numpy(mcb.pcg32_uniforms(rng, 33, S + 1))
        want = mcb.sample(torch.from_numpy(rays).double(), S, lindisp, randomized, u).numpy()
        assert np.abs(t - want).max() <= 8 * 2.0 ** -24 * 6, (S, np.abs(t - want).max())
        assert (np.diff(t, axis=1) >= 0).all() and (t[:, 0] >= 2).all() and (t[:, -1] <= 6).all()


@pytest.mark.parametrize("padding", [0.01, 0.0])
@pytest.mark.parametrize("randomized", [True, False])
def test_resample_f32_within_float64_band(padding, randomized):
    """resample_f32, and mip_cpu_backend.resample (float64), inside resample_band on random, dipping, zero, one-hot and rand^8 rows;
    the fp32 rows sorted and inside [t_0, t_S]."""
    worst = {}
    for S in M.EDGE_S:
        w_hard, kinds = M.resample_rows(S, seed=S, padding=padding)
        g = np.random.default_rng(S)
        w = np.concatenate([w_hard, g.random((8, S)).astype(f32)])
        R = w.shape[0]
        t = M.sample_f32(M.rays_np(R, seed=S), S, False, True, M.pcg_state(S + 50))
        rng = M.pcg_state(S + 100)
        got, cdf = M.resample_f32(t, w, padding, randomized, rng)
        lo, hi = M.resample_band(t, w, padding, randomized, rng)
        u = torch.from_numpy(mcb.pcg32_uniforms(rng, R, S + 1)) if randomized else None
        checks = [("fp32", got)]
        if S > 1:                                              # mip_cpu_backend.resample builds its CDF from cdf[:, :1], empty at S = 1
            checks.append(("float64", mcb.resample(torch.from_numpy(t).double(), torch.from_numpy(w).double(), float(f32(padding)), randomized,
                                                   u).numpy()))
        for name, v in checks:
            r = M.band_ratio(v, lo, hi)
            worst[name] = max(worst.get(name, 0.0), float(r.max()))
            assert (r <= 1).all(), (S, name, np.argwhere(r > 1)[:4], v[r > 1][:4], lo[r > 1][:4], hi[r > 1][:4])
        assert (np.diff(got, axis=1) >= 0).all() and (got >= t[:, :1]).all() and (got <= t[:, -1:]).all()
    print(f"[mip-sampler-bound-cpu] resample band padding={padding} randomized={randomized}: worst position in band {worst}")


def test_the_fp32_cdf_dips_without_padding():
    """The finding the resampling tests are built around: with resample_padding 0, rand^8 weights or weights over 10 decades give fp32
    CDFs that fall by an ulp or a few at a lane boundary (`run` restarts from the lane's scan there); with the configs' 0.01 none do."""
    g = np.random.default_rng(0)
    S = 128
    w = np.concatenate([g.random((500, S)) ** 8, g.random((500, S)) * 10.0 ** g.uniform(-8, 2, (500, S))]).astype(f32)
    d0 = np.diff(M.cdf_f32(w, 0.0), axis=1)
    rows, k = np.nonzero(d0 < 0)
    assert len(set(rows.tolist())) >= 20, len(set(rows.tolist()))
    assert ((k + 1) % 4 == 1).mean() > 0.9                                    # cdf[k + 1] is the first entry a lane writes
    assert (np.abs(d0[d0 < 0]) <= 4 * np.spacing(f32(1))).all()
    assert not (np.diff(M.cdf_f32(w, 0.01), axis=1) < 0).any()
    w_dip, kinds = M.resample_rows(S, seed=1)
    assert kinds.count("dip") == 8
