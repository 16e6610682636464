"""References for the Mip-NeRF sampler kernels of csrc/mip_sampler.cu (no GPU needed).

- sample_f32 / resample_f32: numpy float32 restatements of mip_sample_kernel and mip_resample_kernel, operation for operation.  The
  file is built with -fmad=false and neither kernel calls a transcendental function, so every operation is an IEEE fp32 operation in a
  fixed order and the restatement reproduces the kernels bit for bit: the lanes' sums of 4 weights, the xor butterfly of warp_sum, the
  Hillis-Steele warp_scan, the binary search and the final clamps.  Uniforms are mip_cpu_backend.pcg32_uniforms at index g (S + 1) + j.
- resample_band: where a correct fp32 resampling may place each sample, from a float64 CDF and its error bound.
- composite64 / loss_grad64: the composite forward and the loss backward in float64, each value with a bound on the error of the
  kernels' fp32 evaluation (below), carried through the kernels' expression trees.

Error model (u = 2^-24; every bound is first order, SAFETY = 2 covers the remainder):
- a rounded add / multiply / divide adds u of its result; expf adds 2 ulp (CUDA Programming Guide, maths functions: 4u of the
  result), log1pf 1 ulp (2u); 2^-140 per value covers fp32 subnormal results;
- colour s = 1 / (1 + expf(-x)): s (4u (1 - s) + 2u); c = s k - p with k the kernels' fp32 1 + 2p; the colour derivative
  s (1 - s) k to an absolute bound (1 - s cancels for saturated colours);
- density: x = fl(raw_3 + bias) is taken as the kernel's own fp32 value (one rounding, reproduced exactly); softplus is x itself for
  x > 20 (no error) and log1pf(expf(x)) otherwise: 4u e^x / (1 + e^x) + 2u sigma;
- delta = fl(t_{i+1} - t_i) fl(sqrtf(|d|^2)) against the exact (t_{i+1} - t_i) |d|: 5u of it;
- before_i: lane sums, a warp scan, `scan - local` and serial adds.  Each term passes at most 16 roundings, but `scan - local`
  rounds sums that run to the end of sample i's lane, so the bound is gamma_16 times the optical depth up to that lane's end, plus
  the propagated errors of sd_k, k < i.  T = expf(-before): T expm1(e) + 4u T;
- 1 - expf(-sd) is held to an absolute bound (it cancels for small sd); w = alpha T;
- the sums of rgb, acc and w t_mid: gamma_10 of sum |terms| (4 a lane, a 5-step butterfly, the product), plus the terms' errors;
- distance = clamp(wt / acc, t_0, t_S); where acc's bound reaches acc the bound is the whole [t_0, t_S]; an exact acc of 0 gives t_0;
- loss: the block's fp32 mask sum to gamma_(R / 256 + 9), e = c - target, (mult m) loss / msum and gr = grad_scale ((2 mult) m e / msum)
  in the kernel's order; gc in serial j order; dsd = (T_i expf(-sd_i)) gc_i - (total - upto), the suffix to an ABSOLUTE bound (the
  terms up to i cancel exactly in the kernel's fp32, their rounding does not); then w gr sg and dsd delta dsig.
fp16 outputs are checked by the bracket rn16(d - SAFETY e) <= h <= rn16(d + SAFETY e), which keeps fp16 subnormals: a store that
flushes them fails."""
import numpy as np

from mip_cpu_backend import pcg32_uniforms

f32 = np.float32
U = 2.0 ** -24
SAFETY = 2.0
TINY = 2.0 ** -140
EPS32 = f32(np.finfo(np.float32).eps)
MAX_SAMPLES = 128


def gamma(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------------------- warp primitives
def warp_sum(v):
    """__shfl_xor_sync butterfly over the last axis (32 lanes), fp32; every lane ends with the same value (lane 0's is returned)."""
    v = np.asarray(v, f32).copy()
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(f32)
    return v[..., 0]


def warp_scan(v):
    """Hillis-Steele inclusive prefix sum over the last axis (32 lanes), fp32: v_l += v_(l - o) for lanes l >= o, o = 1, 2, .., 16."""
    v = np.asarray(v, f32).copy()
    for o in (1, 2, 4, 8, 16):
        prev = v.copy()
        v[..., o:] = (prev[..., o:] + prev[..., :-o]).astype(f32)
    return v


def lanes(a, fill=0.0):
    """(R, S, ...) -> (R, 32, 4, ...): sample i = 4 lane + q, padded with `fill` to 128."""
    a = np.asarray(a)
    R, S = a.shape[:2]
    out = np.full((R, MAX_SAMPLES) + a.shape[2:], fill, a.dtype)
    out[:, :S] = a
    return out.reshape((R, 32, 4) + a.shape[2:])


# ---------------------------------------------------------------------------------------------------------------- sampling
def uniforms(rng, R, S):
    """(R, S + 1) float32: draw j of ray g is draw g (S + 1) + j of the pcg32 stream rng = (state, inc); next_float() is exact in fp32."""
    return pcg32_uniforms(rng, R, S + 1).astype(f32)


def fences_f32(rays, S, lindisp):
    near, far = np.asarray(rays, f32)[:, 10:11], np.asarray(rays, f32)[:, 11:12]
    v = (np.arange(S + 1, dtype=f32) / f32(S)).astype(f32)[None]
    if lindisp:
        a = ((f32(1) / near).astype(f32) * (f32(1) - v)).astype(f32)
        b = ((f32(1) / far).astype(f32) * v).astype(f32)
        return (f32(1) / (a + b).astype(f32)).astype(f32)
    return (near + ((far - near).astype(f32) * v).astype(f32)).astype(f32)


def sample_f32(rays, S, lindisp, randomized, rng):
    """mip_sample_kernel: (R, S + 1) float32 fenceposts."""
    F = fences_f32(rays, S, lindisp)
    if not randomized:
        return F
    u = uniforms(rng, F.shape[0], S)
    mids = (f32(0.5) * (F[:, 1:] + F[:, :-1]).astype(f32)).astype(f32)
    lower = np.concatenate([F[:, :1], mids], 1)
    upper = np.concatenate([mids, F[:, -1:]], 1)
    return (lower + ((upper - lower).astype(f32) * u).astype(f32)).astype(f32)


def resample_u_f32(R, S, randomized, rng):
    """The S + 1 sorted u of mip_resample_kernel, (R, S + 1) float32."""
    j = np.arange(S + 1, dtype=f32)[None]
    if randomized:
        s = f32(1) / f32(S + 1)
        r = uniforms(rng, R, S)
        u = ((j * s).astype(f32) + (f32(s - EPS32) * r).astype(f32)).astype(f32)
        return np.fmin(u, f32(f32(1) - EPS32))
    return np.broadcast_to((j * (f32(f32(1) - EPS32) / f32(S))).astype(f32), (R, S + 1)).copy()


def cdf_f32(w, padding):
    """mip_resample_kernel's CDF: (R, S + 1) float32, cdf[0] = 0, cdf[S] = 1, cdf[k] = min(1, run) in between."""
    w = np.asarray(w, f32)
    R, S = w.shape
    pad_f = f32(padding)
    a = w[:, np.maximum(np.arange(S) - 1, 0)]
    c = w[:, np.minimum(np.arange(S) + 1, S - 1)]
    wv = ((f32(0.5) * (np.fmax(a, w) + np.fmax(w, c)).astype(f32)).astype(f32) + pad_f).astype(f32)
    wv = lanes(wv)                                                          # (R, 32, 4), zero past S
    live = lanes(np.ones((R, S), bool), False)

    def lane_sums(x):
        s = np.zeros(x.shape[:2], f32)
        for q in range(4):
            s = (s + x[..., q]).astype(f32)
        return s
    total = warp_sum(lane_sums(wv))
    pad = np.fmax(f32(0), (f32(1e-5) - total).astype(f32))
    wv = np.where(live, (wv + (pad / f32(S)).astype(f32)[:, None, None]).astype(f32), wv)
    local = lane_sums(wv)
    total = (total + pad).astype(f32)
    x = (local / total[:, None]).astype(f32)
    run = (warp_scan(x) - x).astype(f32)
    cdf = np.zeros((R, S + 1), f32)
    flat = np.zeros((R, MAX_SAMPLES), f32)
    for q in range(4):
        run = (run + (wv[..., q] / total[:, None]).astype(f32)).astype(f32)
        flat[:, q::4] = np.fmin(f32(1), run)
    cdf[:, 1:S] = flat[:, :S - 1]
    cdf[:, S] = 1
    return cdf


def invert_f32(t, cdf, u):
    """The binary search (largest k with cdf[k] <= u) and the clamped interpolation of mip_resample_kernel."""
    t, cdf, u = np.asarray(t, f32), np.asarray(cdf, f32), np.asarray(u, f32)
    R, n = u.shape
    S = n - 1
    lo = np.zeros((R, n), np.int64)
    hi = np.full((R, n), S, np.int64)
    rows = np.arange(R)[:, None]
    while True:
        act = hi - lo > 1
        if not act.any():
            break
        mid = (lo + hi) // 2
        le = cdf[rows, mid] <= u
        lo = np.where(act & le, mid, lo)
        hi = np.where(act & ~le, mid, hi)
    c0, c1, t0, t1 = cdf[rows, lo], cdf[rows, lo + 1], t[rows, lo], t[rows, lo + 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.fmin(np.fmax(((u - c0).astype(f32) / (c1 - c0).astype(f32)).astype(f32), f32(0)), f32(1))
    return np.fmin(np.fmax((t0 + (f * (t1 - t0).astype(f32)).astype(f32)).astype(f32), t0), t1)


def resample_f32(t, w, padding, randomized, rng):
    """mip_resample_kernel: ((R, S + 1) float32 resampled fenceposts, its (R, S + 1) float32 CDF)."""
    t = np.asarray(t, f32)
    R, S = t.shape[0], t.shape[1] - 1
    cdf = cdf_f32(w, padding)
    return invert_f32(t, cdf, resample_u_f32(R, S, randomized, rng)), cdf


# ---------------------------------------------------------------------------------------------------------------- resampling band
def cdf64(w, padding):
    """(cdf (R, S + 1) float64 with the kernels' fp32 constants, its error bound on the fp32 kernel's CDF)."""
    w = np.asarray(w, f32).astype(np.float64)
    R, S = w.shape
    wp = np.concatenate([w[:, :1], w, w[:, -1:]], 1)
    wm = np.maximum(wp[:, :-1], wp[:, 1:])
    wv = 0.5 * (wm[:, :-1] + wm[:, 1:]) + float(f32(padding))
    ws = wv.sum(1, keepdims=True)
    pad = np.maximum(float(f32(1e-5)) - ws, 0)
    wv = wv + pad / S
    ws = ws + pad
    c = np.minimum(np.cumsum(wv / ws, 1)[:, :-1], 1)
    cdf = np.concatenate([np.zeros((R, 1)), c, np.ones((R, 1))], 1)
    # relative errors: a blurred weight 4u, a lane sum 3u, the butterfly 5u and + pad u, the quotients u, the scan 5u, scan - x u,
    # the lane's serial adds 4u: 75u of the CDF at the end of the lane that writes cdf[k] (entry k is written by lane (k - 1) / 4),
    # and, with the 1e-5 padding, 32u absolute for its spread
    k = np.arange(1, S)
    end = np.minimum(4 * ((k - 1) // 4 + 1), S)
    full = np.concatenate([np.zeros((R, 1)), np.cumsum(wv / ws, 1)], 1)
    err = np.zeros_like(cdf)
    err[:, 1:S] = 75 * U * full[:, end] + np.where(pad > 0, 32 * U, 0.0)
    return cdf, err


def resample_u64(R, S, randomized, rng):
    """(u float64 as the reference computes it, bound on the kernel's fp32 u)."""
    n = S + 1
    eps = float(EPS32)
    j = np.arange(n, dtype=np.float64)[None]
    if randomized:
        s = 1.0 / n
        u = np.minimum(j * s + (s - eps) * pcg32_uniforms(rng, R, n), 1 - eps)
        return u, 6 * U * u + TINY
    u = np.broadcast_to(np.linspace(0.0, 1 - eps, n), (R, n)).copy()
    return u, 3 * U * u


def _first_at_least(t, c, v):
    """min {x : C(x) >= v} of the piecewise-linear C through (t_k, c_k), for each v (row-wise); t_0 if c_0 >= v."""
    R, n = v.shape
    ge = c[:, :, None] >= v[:, None, :]                                       # (R, knots, n)
    k = np.where(ge.any(1), ge.argmax(1), n - 1)
    rows = np.arange(R)[:, None]
    km = np.maximum(k - 1, 0)
    c0, c1, t0, t1 = c[rows, km], c[rows, k], t[rows, km], t[rows, k]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.clip(np.nan_to_num((v - c0) / (c1 - c0), nan=1.0, posinf=1.0, neginf=0.0), 0, 1)
    return np.where(k == 0, t[:, :1], t0 + f * (t1 - t0))


def _last_at_most(t, c, v):
    """max {x : C(x) <= v}; t_S if c_S <= v."""
    R, n = v.shape
    le = c[:, :, None] <= v[:, None, :]
    S = c.shape[1] - 1
    k = np.where(le.any(1), S - le[:, ::-1].argmax(1), 0)
    rows = np.arange(R)[:, None]
    kp = np.minimum(k + 1, S)
    c0, c1, t0, t1 = c[rows, k], c[rows, kp], t[rows, k], t[rows, kp]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.clip(np.nan_to_num((v - c0) / (c1 - c0), nan=0.0, posinf=1.0, neginf=0.0), 0, 1)
    return np.where(k == S, t[:, S:], t0 + f * (t1 - t0))


def resample_band(t, w, padding, randomized, rng):
    """(lo, hi) (R, S + 1) float64: a correct fp32 resampling puts sample j between the inverse of the float64 CDF plus its bound at
    u - du and the inverse of the CDF minus its bound at u + du (generalised inverses: no monotone fp32 CDF is assumed); widened by
    the fp32 interpolation t0 + f (t1 - t0) (4u of |t|).  Tight where the pdf is not tiny, the flat stretch where it is."""
    t64 = np.asarray(t, f32).astype(np.float64)
    R, S = t64.shape[0], t64.shape[1] - 1
    c, e = cdf64(w, padding)
    u, du = resample_u64(R, S, randomized, rng)
    e = SAFETY * e
    du = SAFETY * du
    lo = _first_at_least(t64, c + e, u - du)
    hi = _last_at_most(t64, c - e, u + du)
    slack = 4 * U * np.maximum(np.abs(lo), np.abs(hi))
    return lo - slack, hi + slack


def band_ratio(got, lo, hi):
    """0 at the band's centre, 1 at its edges, > 1 outside (NaN outside)."""
    g = np.asarray(got, np.float64)
    mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(half > 0, np.abs(g - mid) / half, np.where(g == mid, 0.0, np.inf))
    return np.where(np.isnan(g), np.inf, r)


# ---------------------------------------------------------------------------------------------------------------- composite
def _logistic(x):
    """(exact 1 / (1 + e^-x), bound of the fp32 1.f / (1.f + expf(-x)))."""
    with np.errstate(over="ignore"):
        s = 1.0 / (1.0 + np.exp(-x))
    return s, s * (4 * U * (1 - s) + 2 * U) + 2.0 ** -126


def _expm(x, e):
    """(exp(-x), bound of expf(-x~)) for |x~ - x| <= e."""
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.exp(-x)
        e = np.where(v > 0, v * np.expm1(e) + 4 * U * v * np.exp(e), 0.0)
    return v, e + 2.0 ** -148


def forward64(raw, t, rays, p, bias):
    """Per-sample (R, S) float64 values and bounds of ray_forward.  raw (R, S, 4) fp16 or fp32, t (R, S + 1) fp32, rays (R, 12) fp32."""
    raw = np.asarray(raw)
    R, S = raw.shape[:2]
    r64 = raw.astype(np.float64)
    t64 = np.asarray(t, f32).astype(np.float64)
    p32 = f32(p)
    k = float(f32(f32(1) + f32(f32(2) * p32)))
    s, es = _logistic(r64[..., :3])
    c = s * k - float(p32)
    ec = k * es + U * np.abs(s * k) + U * np.abs(c) + TINY
    one_s, e1s = 1 - s, es                                                  # fl(1 - s~): + u |1 - s|
    e1s = e1s + U * np.abs(one_s)
    ss = s * one_s
    ess = es * np.abs(one_s) + np.abs(s) * e1s + U * ss
    sg = ss * k
    esg = k * ess + U * sg + TINY
    x32 = (raw[..., 3].astype(f32) + f32(bias)).astype(f32)                 # the kernel's x, one rounding
    x = x32.astype(np.float64)
    big = x32 > f32(20)
    with np.errstate(over="ignore"):
        ex = np.exp(np.where(big, 0.0, x))
    sigma = np.where(big, x, np.log1p(ex))
    esig = np.where(big, 0.0, 4 * U * ex / (1 + ex) + 2 * U * sigma + 2.0 ** -148)
    dsig, edsig = _logistic(x)
    d = np.asarray(rays, f32)[:, 3:6].astype(np.float64)
    dn = np.sqrt((d * d).sum(1))[:, None]
    dt = t64[:, 1:] - t64[:, :-1]
    delta = dt * dn
    edelta = 5 * U * np.abs(delta) + TINY
    sd = sigma * delta
    esd = sigma * edelta + np.abs(delta) * esig + U * np.abs(sd) + TINY
    # before: the exact exclusive prefix; its bound: gamma_16 of the optical depth to the end of the sample's lane, + propagated errors
    before = np.concatenate([np.zeros((R, 1)), np.cumsum(sd, 1)[:, :-1]], 1)
    prop = np.concatenate([np.zeros((R, 1)), np.cumsum(esd, 1)[:, :-1]], 1)
    cum = np.cumsum(np.abs(sd) + esd, 1)
    end = np.minimum(4 * (np.arange(S) // 4 + 1), S) - 1
    ebefore = gamma(16) * cum[:, end] + prop + TINY
    T, eT = _expm(before, ebefore)
    A, eA = _expm(sd, esd)
    with np.errstate(over="ignore"):
        al = -np.expm1(-sd)
    eal = eA + U * al
    w = al * T
    ew = al * eT + T * eal + eal * eT + U * w + TINY
    tm = 0.5 * (t64[:, 1:] + t64[:, :-1])
    etm = U * np.abs(tm)
    return dict(c=c, ec=ec, sg=sg, esg=esg, dsig=dsig, edsig=edsig, delta=delta, edelta=edelta, sd=sd, esd=esd, T=T, eT=eT, A=A, eA=eA,
                w=w, ew=ew, tm=tm, etm=etm, t64=t64)


def _sum(terms, errs, n=10):
    """A kernel sum over samples (lanes of 4, then the butterfly): value and bound."""
    return terms.sum(1), errs.sum(1) + gamma(n) * np.abs(terms).sum(1) + TINY


def composite64(raw, t, rays, p, bias, white):
    """mip_composite_fwd_kernel in float64: dict of (value, bound) for rgb (R, 3), acc (R,), distance (R,), weights (R, S), and the
    per-sample quantities (key `f`) the loss uses."""
    f = forward64(raw, t, rays, p, bias)
    w, ew, c, ec = f["w"], f["ew"], f["c"], f["ec"]
    acc, eacc = _sum(w, ew)
    rgb = np.empty((w.shape[0], 3))
    ergb = np.empty_like(rgb)
    for j in range(3):
        rgb[:, j], ergb[:, j] = _sum(w * c[..., j], np.abs(w) * ec[..., j] + np.abs(c[..., j]) * ew + ew * ec[..., j])
        if white:
            rgb[:, j] = rgb[:, j] + (1 - acc)
            ergb[:, j] = ergb[:, j] + eacc + U * np.abs(1 - acc) + U * np.abs(rgb[:, j])
    wt, ewt = _sum(w * f["tm"], np.abs(w) * f["etm"] + np.abs(f["tm"]) * ew)
    t64 = f["t64"]
    t0, tS = t64[:, 0], t64[:, -1]
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.where(acc > 0, wt / acc, t0)
        ed = (ewt + np.abs(d) * SAFETY * eacc) / (acc - SAFETY * eacc) + U * np.abs(d)
    dist = np.minimum(np.maximum(d, t0), tS)
    edist = np.where(acc == 0, 0.0, np.where(acc > 2 * SAFETY * eacc, ed, tS - t0))
    return dict(rgb=(rgb, ergb), acc=(acc, eacc), dist=(dist, edist), w=(w, ew), f=f)


def mask_sum(mask, R):
    """(the exact mask sum, bound of the block's fp32 sum: a serial stride-256 sum, then an 8-level tree); f32(R) without a mask."""
    if mask is None:
        return float(f32(R)), 0.0
    m = np.asarray(mask, f32).astype(np.float64)
    return m.sum(), gamma(-(-R // 256) + 9) * np.abs(m).sum() + TINY


def loss_grad64(raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale):
    """mip_loss_bwd_kernel in float64 over the 2R rays (coarse, then fine): (rgb, bound) (2R, 3), (loss, bound) (2R,),
    (d(raw), bound) (2R, S, 4).  rays / target / mask are those of the R rays."""
    rays = np.asarray(rays, f32)
    R = rays.shape[0]
    comp = composite64(raw, t, np.concatenate([rays, rays]), p, bias, white)
    f = comp["f"]
    rgb, ergb = comp["rgb"]
    msum, emsum = mask_sum(mask, R)
    m = np.ones(R) if mask is None else np.asarray(mask, f32).astype(np.float64)
    m = np.concatenate([m, m])
    mult = np.concatenate([np.full(R, float(f32(coarse_mult))), np.ones(R)])
    gs = float(f32(grad_scale))
    tg = np.asarray(target, f32).astype(np.float64)
    tg = np.concatenate([tg, tg])
    e = rgb - tg
    ee = ergb + U * np.abs(e)
    sq = e * e
    esq = 2 * np.abs(e) * ee + ee * ee + U * sq
    loss = sq.sum(1)
    eloss = esq.sum(1) + gamma(2) * sq.sum(1)
    a = mult * m
    lv = a * loss / msum
    elv = np.abs(a / msum) * eloss + np.abs(lv) * (emsum / msum + 3 * U) + TINY
    coef = (gs * 2 * mult * m / msum)[:, None]
    gr = coef * e
    egr = np.abs(gr) * (4 * U + emsum / msum) + np.abs(coef) * ee + TINY
    c, ec = f["c"], f["ec"]
    cb = c - (1.0 if white else 0.0)
    ecb = ec + (U * np.abs(cb) if white else 0.0)
    terms = gr[:, None, :] * cb
    eterms = np.abs(gr)[:, None, :] * ecb + np.abs(cb) * egr[:, None, :] + U * np.abs(terms)
    gc = terms.sum(2)
    egc = eterms.sum(2) + gamma(2) * np.abs(terms).sum(2) + TINY
    w, ew = f["w"], f["ew"]
    wgc = w * gc
    ewgc = np.abs(w) * egc + np.abs(gc) * ew + U * np.abs(wgc)
    suffix = np.cumsum(wgc[:, ::-1], 1)[:, ::-1] - wgc                    # sum_(k > i) w_k gc_k
    eprop = np.cumsum(ewgc[:, ::-1], 1)[:, ::-1] - ewgc
    esuffix = 2 * gamma(16) * np.abs(wgc).sum(1, keepdims=True) + eprop + U * np.abs(suffix) + TINY
    TA = f["T"] * f["A"]
    eTA = f["T"] * f["eA"] + f["A"] * f["eT"] + f["eA"] * f["eT"] + U * TA + TINY
    first = TA * gc
    efirst = TA * egc + np.abs(gc) * eTA + U * np.abs(first)
    dsd = first - suffix
    edsd = efirst + esuffix + U * np.abs(dsd) + TINY
    R2, S = w.shape
    d = np.empty((R2, S, 4))
    ed = np.empty_like(d)
    sg, esg = f["sg"], f["esg"]
    for j in range(3):
        v = w * gr[:, None, j] * sg[..., j]
        d[..., j] = v
        ed[..., j] = (np.abs(gr[:, None, j] * sg[..., j]) * ew + np.abs(w * sg[..., j]) * egr[:, None, j] + np.abs(w * gr[:, None, j]) * esg[..., j]
                      + 2 * U * np.abs(v) + TINY)
    delta, edelta, dsig, edsig = f["delta"], f["edelta"], f["dsig"], f["edsig"]
    v = dsd * delta * dsig
    d[..., 3] = v
    ed[..., 3] = (np.abs(delta * dsig) * edsd + np.abs(dsd * dsig) * edelta + np.abs(dsd * delta) * edsig + 2 * U * np.abs(v) + TINY)
    return (rgb, ergb), (lv, elv), (d, ed)


# ---------------------------------------------------------------------------------------------------------------- checks
def ratio32(got, exact, err):
    """|got - exact| / (SAFETY err); an entry with a zero bound must be exact; NaN fails."""
    g = np.asarray(got, np.float64)
    dd = np.abs(g - exact)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, dd / (SAFETY * err), np.where(dd == 0, 0.0, np.inf))
    return np.where(np.isnan(dd), np.inf, r)


def check16(got, exact, err):
    """(ok, ratio) of fp16 values: ok where rn16(exact - SAFETY err) <= got <= rn16(exact + SAFETY err); the ratio (for the report) is
    |got - exact| over SAFETY err plus half the fp16 spacing at exact."""
    with np.errstate(over="ignore", invalid="ignore"):
        lo = (exact - SAFETY * err).astype(np.float16).astype(np.float64)
        hi = (exact + SAFETY * err).astype(np.float16).astype(np.float64)
        g = np.asarray(got).astype(np.float64)
        ok = (g >= lo) & (g <= hi)
        sp = np.spacing(np.abs(exact).astype(np.float16)).astype(np.float64)
        r = np.abs(g - exact) / (SAFETY * err + 0.5 * sp)
    return ok, np.where(ok, np.nan_to_num(r, nan=0.0, posinf=0.0), np.inf)


class Tally:
    """Worst ratio per quantity, and a description of the first failing entry of each quantity."""

    def __init__(self):
        self.worst, self.fails = {}, []

    def note(self, name, r):
        self.worst[name] = max(self.worst.get(name, 0.0), float(np.max(r)) if np.size(r) else 0.0)

    def bound(self, name, got, value, err, tag=""):
        got = np.asarray(got)
        if got.dtype == np.float16:
            ok, r = check16(got, value, err)
        else:
            r = ratio32(got, value, err)
            ok = r <= 1
        self.note(name, r)
        if not ok.all():
            i = np.unravel_index(np.argmax(~ok), ok.shape)
            self.fails.append(f"{tag}{name}: {int((~ok).sum())} entries outside the bound, first at {tuple(int(x) for x in i)}: got "
                              f"{got[i]!r}, exact {value[i]!r}, bound {SAFETY * err[i]!r}")
        return ok

    def exact(self, name, ok, tag=""):
        ok = np.asarray(ok)
        if not ok.all():
            i = np.unravel_index(np.argmax(~ok), ok.shape)
            self.fails.append(f"{tag}{name}: {int((~ok).sum())} entries differ, first at {tuple(int(x) for x in i)}")

    def report(self):
        return ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items()))


def check_composite(tally, got, raw, t, rays, p, bias, white, tag=""):
    """got = (rgb, acc, dist, w) of mip_composite_fwd; every entry within composite64's bound."""
    ex = composite64(raw, t, rays, p, bias, white)
    for name, g in zip(("rgb", "acc", "dist", "w"), got):
        if g is not None:
            tally.bound(f"composite {name}", g, *ex[name], tag=tag)
    return ex


def check_loss(tally, got, raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale, tag=""):
    """got = (rgb (2R, 3), loss (2R,), draw (2R S, 4)) of mip_composite_loss_bwd."""
    (rgb, erg), (lv, el), (d, ed) = loss_grad64(raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale)
    tally.bound("loss rgb", got[0], rgb, erg, tag)
    tally.bound("loss", got[1], lv, el, tag)
    dr = np.asarray(got[2]).reshape(d.shape)
    dn = np.dtype(dr.dtype).name
    tally.bound(f"d(raw) colour {dn}", dr[..., :3], d[..., :3], ed[..., :3], tag)
    tally.bound(f"d(raw) density {dn}", dr[..., 3], d[..., 3], ed[..., 3], tag)
    return d


# ---------------------------------------------------------------------------------------------------------------- batches
EDGE_S = [1, 2, 3, 4, 5, 31, 32, 33, 127, 128]
EDGE_R = [1, 7, 8, 9, 257]


def rays_np(R, seed, d_max=2.0):
    """(R, 12) float32 rays towards the origin, |d| in [1, d_max], radii of four resolutions, near 2, far 6."""
    g = np.random.default_rng(seed)
    o = (g.random((R, 3)) - 0.5) * 8
    d = -o + g.normal(0, 0.3, (R, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    v = d.copy()
    d = d * (1 + (d_max - 1) * g.random((R, 1)))
    radius = 1.2e-3 * 2.0 ** (np.arange(R) % 4)[:, None]
    return np.concatenate([o, d, v, radius, np.full((R, 1), 2.0), np.full((R, 1), 6.0)], 1).astype(f32)


def pcg_state(seed):
    """A pcg32 (state, inc) pair without the library: any odd increment gives a full-period stream."""
    g = np.random.default_rng(seed)
    return np.array([int(g.integers(0, 2 ** 63)) * 2 + 1, int(g.integers(0, 2 ** 62)) * 2 + 1], np.uint64)


def edge_batch(R, S, seed):
    """Both levels of R rays of S samples: dict(rays (R, 12), t (2R, S + 1), raw (2R, S, 4) float32 values exact in fp16, target,
    masks).  Densities spread the ray's optical depth from transparent to opaque; every third ray is fully transparent on one level."""
    g = np.random.default_rng(seed)
    rays = rays_np(R, seed)
    t = np.concatenate([sample_f32(rays, S, False, True, pcg_state(seed)), sample_f32(rays, S, True, True, pcg_state(seed + 1))])
    raw = np.empty((2 * R, S, 4), f32)
    raw[..., :3] = g.normal(0, 2.5, (2 * R, S, 3))
    tau = 10.0 ** g.uniform(-2, 1.5, (2 * R, 1))                                # optical depth of the ray
    dt = (t[:, 1:] - t[:, :-1]).astype(np.float64) * 2.0 + 1e-6
    raw[..., 3] = np.log(np.expm1(np.clip(tau / S / dt, 1e-30, 30))) + 1 + g.normal(0, 1.0, (2 * R, S))
    raw[(np.arange(2 * R) % 3 == 2), :, 3] = -1e4                              # sigma = 0: acc 0, distance t_0
    raw = raw.astype(np.float16).astype(f32)
    target = g.random((R, 3)).astype(f32)
    zeros = ((g.random(R) > 0.3) * g.choice([1.0, 4.0, 16.0, 64.0], R)).astype(f32)    # multicam's lossmult, with zeros
    zeros[0], zeros[-1] = 0.0, 4.0
    return dict(rays=rays, t=t, raw=raw, target=target, masks=[None, zeros])


def adversarial_batch(seed=900, S=128, fp16=True):
    """Rows where the composite goes wrong first: x = raw_3 + bias at 20 and one fp32 (fp16) ulp either side, saturated colours, a first
    sample that takes T to 0 or to a subnormal, transparent rays, zero-length intervals and |d| up to 2.  bias = -1."""
    R = 48
    g = np.random.default_rng(seed)
    b = edge_batch(R, S, seed)
    raw, t, rays = b["raw"], b["t"], b["rays"]
    up = (lambda v: np.float16(v).item() + 2.0 ** -6) if fp16 else (lambda v: float(np.nextafter(f32(v), f32(99))))
    dn = (lambda v: np.float16(v).item() - 2.0 ** -6) if fp16 else (lambda v: float(np.nextafter(f32(v), f32(-99))))
    for r in range(0, 2 * R, 5):
        k = g.integers(0, S, 6)
        raw[r, k, 3] = [21.0, up(21.0), dn(21.0), 21.0, up(21.0), dn(21.0)]
    for r in range(1, 2 * R, 5):
        k = g.random((S, 3)) < 0.3
        raw[r, :, :3][k] = g.choice([30.0, -30.0, 65504.0, -65504.0], int(k.sum()))
    dt = (t[:, 1:] - t[:, :-1]).astype(np.float64) * np.linalg.norm(np.concatenate([rays, rays])[:, 3:6], axis=1)[:, None]
    for r in range(2, 2 * R, 5):                                                # T underflows to 0 (sd ~ 2000) or a subnormal (sd ~ 90)
        raw[r, 0, 3] = 65504.0 if r % 2 else np.float16(90.0 / dt[r, 0] + 1).item()
    for r in range(3, 2 * R, 5):
        raw[r, :, 3] = -1e4
    for r in range(4, 2 * R, 5):                                                # zero-length intervals, as a peaked resample leaves
        k = np.sort(g.choice(S, min(S, 8), replace=False))
        for kk in k:
            t[r, kk + 1] = t[r, kk]
        t[r] = np.maximum.accumulate(t[r])
    raw = raw.astype(np.float16).astype(f32) if fp16 else raw
    return dict(b, raw=raw, t=t)


def resample_rows(S, seed, padding=0.0, n=8):
    """(w (n_rows, S) float32, kinds) of resampling's hard rows: rows whose fp32 CDF dips (found by search), all-zero rows, one-hot
    rows and rand^8 rows."""
    g = np.random.default_rng(seed)
    cand = np.concatenate([(g.random((2000, S)) ** 8), g.random((2000, S)) * 10.0 ** g.uniform(-8, 2, (2000, S))]).astype(f32)
    dips = cand[(np.diff(cdf_f32(cand, padding), axis=1) < 0).any(1)][:n]
    one_hot = np.zeros((n, S), f32)
    one_hot[np.arange(n), g.integers(0, S, n)] = g.random(n).astype(f32) + f32(0.5)
    rows = [dips, np.zeros((2, S), f32), one_hot, (g.random((n, S)) ** 8).astype(f32)]
    kinds = ["dip"] * len(dips) + ["zero"] * 2 + ["one-hot"] * n + ["rand^8"] * n
    return np.concatenate(rows), kinds
