"""References for the NGP optimizer tail of csrc/optimizer.cu (no GPU needed): ngp_adam_ema and ngp_train_sweep both end in adam_one
(csrc/train_common.cuh), and the sweep forms its table gradient from the fused backward's int64 fixed-point sums.

- Hyper: the fp32 hyper-parameters the kernels receive, and step_size, debias_old and debias_new formed in double as make_adam_args
  forms them (the kernels get them rounded to fp32).
- adam_ema64: adam_one in float64 from the kernel's own input state, with a bound on every entry of m, v and master.  Every call
  starts from what the kernel read, so errors do not compound over steps.
- adam_one_f32: adam_one in numpy float32, operation for operation, and the mutants the bound must reject.
- fx_grad64: the fp16 gradient of one fixed-point sum, rn16(rn32(q) 2^-32), computed exactly on the host.
- make_state / fx_sums: the input distributions of the tests.

Error model (u = 2^-24).  adam_one's rounded operations, in their order:
  g' = g grad_scale;  t1 = (1 - b1) g';  m1 = fma(b1, m, t1);  t2 = (1 - b2) g';  t3 = t2 g';  v1 = fma(b2, v, t3);
  s = sqrtf(v1);  d = s + eps;  n = m1 step_size;  q = n / d;  p = master - q;
  a = decay master;  b = a debias_old;  c = fma(1 - decay, p, b);  master1 = c debias_new.
Each adds u of its result, and 2^-149 where the result can be subnormal; sqrtf and the quotient are correctly rounded (optimizer.cu is
built without fast-math).  1 - b1, 1 - b2 and 1 - decay are exact in fp32 for the values used here (Sterbenz; Hyper asserts it), and
step_size, debias_old and debias_new add u each for their rounding to fp32.  The errors of g', m1 and v1 are carried into the update:
|sqrt(v1~) - sqrt(v1)| <= min(e_v / sqrt(v1), sqrt(e_v)) and |n~ / d~ - n / d| <= (e_n + |q| e_d) / (d - e_d).  The bound is a worst
case with its second-order terms kept, not an estimate: the tests hold every entry to it with no safety factor."""
import math

import numpy as np
import torch

U = 2.0 ** -24
TINY = 2.0 ** -149
FX_INV = 2.0 ** -32
f32 = np.float32
MUTANTS = ["debias-old-at-step-1", "swap-decay", "lr-for-step-size", "swap-betas", "eps-in-sqrt", "grad-scale-twice", "ema-reads-p"]


def _xp(a):
    return torch if isinstance(a, torch.Tensor) else np


def expdecay_lr(step, base_lr=0.1, decay_start=20000, decay_interval=10000, decay_base=0.33):
    """The learning rate of Adam step `step` (1-based) under lego_cfg's ExpDecay (optims/expdecay.py): the factor is decided from the
    0-based step count before it is incremented and accumulates one product per boundary reached"""
    f = 1
    for k in range(decay_start, step, decay_interval):
        f *= decay_base
    return base_lr * f


class Hyper:
    """The arguments of one ngp_adam_ema / ngp_train_sweep call, as the kernel receives them."""

    def __init__(self, lr, step, b1=0.9, b2=0.99, eps=1e-15, decay=0.95, grad_scale=1.0):
        self.lr, self.b1, self.b2, self.eps, self.decay, self.grad_scale = (float(f32(x)) for x in (lr, b1, b2, eps, decay, grad_scale))
        self.step = int(step)
        assert self.step >= 1
        for b in (self.b1, self.b2, self.decay):
            assert float(f32(1) - f32(b)) == 1.0 - b, "1 - b must be exact in fp32 for this bound"
        n1, n2 = 1.0 - self.b1 ** self.step, 1.0 - self.b2 ** self.step
        self.step_size = self.lr * math.sqrt(n2) / n1
        self.debias_old = 1.0 - self.decay ** (self.step - 1.0)
        self.debias_new = 1.0 / (1.0 - self.decay ** self.step)

    def __repr__(self):
        return f"Hyper(lr={self.lr:.6g}, step={self.step}, decay={self.decay:g}, grad_scale={self.grad_scale:.6g})"


def adam_ema64(g, m, v, master, h, full=False):
    """(m1, e_m, v1, e_v, master1, e_master): one adam_one of every entry in float64 from the kernel's input g (the gradient before
    grad_scale), m, v and master (float64 arrays or tensors), with the bound of each output.  full=True also returns (p, e_p), the Adam
    update before the EMA."""
    xp = _xp(g)
    c1, c2, cd = 1.0 - h.b1, 1.0 - h.b2, 1.0 - h.decay
    G = g * h.grad_scale
    aG = abs(G)
    eg = U * aG + TINY
    # m1 = fma(b1, m, fl((1 - b1) g'))
    M1 = h.b1 * m + c1 * G
    et1 = c1 * eg + U * c1 * (aG + eg) + TINY
    em = (1 + U) * et1 + U * abs(M1) + TINY
    # v1 = fma(b2, v, fl(fl((1 - b2) g') g'))
    V1 = h.b2 * v + c2 * G * G
    et2 = c2 * eg + U * c2 * (aG + eg) + TINY
    e23 = et2 * (aG + eg) + c2 * aG * eg
    et3 = e23 + U * (c2 * G * G + e23) + TINY
    ev = (1 + U) * et3 + U * V1 + TINY
    # q = fl(fl(m1 step_size) / fl(sqrtf(v1) + eps))
    S = xp.sqrt(V1)
    es = xp.minimum(ev / xp.maximum(S, xp.full_like(S, 1e-300)), xp.sqrt(ev))
    es = es + U * (S + es)
    D = S + h.eps
    ed = es + U * (D + es)
    N = M1 * h.step_size
    en = em * h.step_size * (1 + U) + U * abs(M1) * h.step_size
    en = en + U * (abs(N) + en) + TINY
    Q = N / D
    lo = D - ed
    eq = xp.where(lo > 0, (en + abs(Q) * ed) / xp.where(lo > 0, lo, xp.ones_like(lo)), xp.full_like(lo, math.inf))
    eq = eq + U * (abs(Q) + eq) + TINY
    P = master - Q
    ep = eq + U * (abs(P) + eq) + TINY
    # master1 = fl(fma(1 - decay, p, fl(fl(decay master) debias_old)) debias_new)
    A = h.decay * master
    ea = U * abs(A) + TINY
    B = A * h.debias_old
    eb = ea * h.debias_old * (1 + U) + U * abs(A) * h.debias_old
    eb = eb + U * (abs(B) + eb) + TINY
    C = cd * P + B
    ec = cd * ep + eb
    ec = ec + U * (abs(C) + ec) + TINY
    MS = C * h.debias_new
    ems = ec * h.debias_new * (1 + U) + U * abs(C) * h.debias_new
    ems = ems + U * (abs(MS) + ems) + TINY
    out = (M1, em, V1, ev, MS, ems)
    return out + (P, ep) if full else out


def ratio(got, exact, err):
    """|got - exact| / err per entry (float64); NaN or an infinite value in got gives inf."""
    xp = _xp(exact)
    d = abs(got - exact)
    r = d / err
    return xp.where(xp.isfinite(d), r, xp.full_like(r, math.inf))


# ------------------------------------------------------------------------------------------------------------ fp32 emulation
def _fma32(a, b, c):
    """fma in float32 through float64: a b is exact in double; the add rounds once in double before the rounding to fp32 (a double
    rounding that can differ from the fused result only where the double sum lands on an fp32 midpoint)."""
    return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def adam_one_f32(g, m, v, master, h, mutant=None):
    """adam_one on float32 arrays -> (m1, v1, master1); `mutant` names one of MUTANTS: a plausible slip in the kernel's arithmetic."""
    assert mutant in (None, *MUTANTS)
    g, m, v, master = (np.asarray(x, f32) for x in (g, m, v, master))
    b1, b2, eps, d, gs = (f32(x) for x in (h.b1, h.b2, h.eps, h.decay, h.grad_scale))
    ss, dbo, dbn = f32(h.step_size), f32(h.debias_old), f32(h.debias_new)
    if mutant == "swap-betas":
        b1, b2 = b2, b1
    if mutant == "lr-for-step-size":
        ss = f32(h.lr)
    if mutant == "debias-old-at-step-1" and h.step == 1:
        dbo = f32(1)
    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        g = g * gs
        if mutant == "grad-scale-twice":
            g = g * gs
        m1 = _fma32(b1, m, (f32(1) - b1) * g)
        v1 = _fma32(b2, v, ((f32(1) - b2) * g) * g)
        den = np.sqrt(v1 + eps) if mutant == "eps-in-sqrt" else np.sqrt(v1) + eps
        p = master - (m1 * ss) / den
        hist = (d * (p if mutant == "ema-reads-p" else master)) * dbo
        ms = _fma32(d, p, (f32(1) - d) * master * dbo) if mutant == "swap-decay" else _fma32(f32(1) - d, p, hist)
        ms = ms * dbn
    return m1, v1, ms


# ------------------------------------------------------------------------------------------------------------ fixed point
def fx_grad64(q):
    """The fp16 gradient (as float64) the training sweep and the flush form from int64 fixed-point sums q in units of 2^-32:
    rn16(rn32(q) 2^-32).  numpy's int64 -> float32 rounds to nearest, the scaling is exact and float32 -> float16 is correctly rounded,
    so this is exact.  It is also checked to lie within half an fp16 ulp of the exact q 2^-32 (the subnormal spacing below 2^-14), with
    one part in 2^13 to spare for the double rounding."""
    q = np.asarray(q, np.int64)
    assert np.abs(q).max(initial=0) < 2 ** 53
    h = (q.astype(f32) * f32(FX_INV)).astype(np.float16).astype(np.float64)
    x = q.astype(np.float64) * FX_INV
    assert np.isfinite(h).all(), "a sum rounds past 65504"
    e = np.frexp(np.abs(x))[1] - 1
    half = np.ldexp(1.0, np.maximum(e, -14) - 11)
    bad = np.abs(h - x) > half * (1 + 2.0 ** -13)
    assert not bad.any(), f"rn16(rn32(q) 2^-32) is off by more than half an fp16 ulp at q = {q[bad][:4].tolist()}"
    return h


def fx_sums(n_entries, rng):
    """(n_entries, 2) int64 sums of the shapes a backward leaves: zero (a quarter of the features, so that entries with one zero feature
    and one nonzero occur), +-1, more than 24 significant bits (the fp32 step rounds), just inside the fp16 range, fp16 subnormals
    including exact rounding ties (q = (2k + 1) 2^7, half the subnormal spacing 2^8) and log-uniform magnitudes."""
    n = 2 * n_entries
    kind = rng.integers(0, 8, n)
    sign = np.where(rng.random(n) < 0.5, -1, 1).astype(np.int64)
    mag = np.zeros(n, np.int64)
    mag[kind == 1] = 1
    k = kind == 2
    mag[k] = rng.integers(1 << 30, 1 << 45, int(k.sum())) | 1                                  # odd: more than 24 significant bits
    k = kind == 3
    mag[k] = rng.integers(65000 << 32, (65510 << 32) + 1, int(k.sum()))
    k = kind == 4
    mag[k] = rng.integers(1, 1 << 18, int(k.sum()))
    k = kind == 5
    mag[k] = (2 * rng.integers(0, 1 << 9, int(k.sum())) + 1) * 128 + rng.integers(-1, 2, int(k.sum()))
    k = kind >= 6
    mag[k] = np.exp2(rng.uniform(0, 46, int(k.sum()))).astype(np.int64)
    return (sign * mag).reshape(n_entries, 2)


# ------------------------------------------------------------------------------------------------------------ inputs
def make_state(n, param_fp16, grad_dtype, seed, device="cpu"):
    """(g, m, v, master) for n parameters as torch tensors (g in grad_dtype, the rest fp32):
    - v >= 0 log-uniform over 10^-40 .. 10^4 (fp32 subnormals included), an eighth exact zeros;
    - m of either sign, up to sqrt(v);
    - master up to 0.1 in magnitude (uniform, a quarter log-uniform down to 1e-8, a few exact zeros), rounded to fp16 when the parameter
      is fp16;
    - g log-uniform over 10^-9 .. 65504 of either sign, an eighth exact zeros, a sixteenth fp16 subnormals, a sixteenth +-65504, and for
      fp32 gradients a sixteenth fp32 subnormals;
    - one entry in 32 has g = m = v = 0."""
    gen = torch.Generator(device=device).manual_seed(seed)

    def uni(lo=0.0, hi=1.0):
        return torch.rand(n, generator=gen, device=device, dtype=torch.float64) * (hi - lo) + lo

    def sign():
        return torch.where(uni() < 0.5, -1.0, 1.0).to(torch.float64)

    v = torch.exp2(uni(-40, 4) * math.log2(10))
    v = torch.where(uni() < 0.125, 0.0, v).float()
    m = (sign() * uni() * v.double().sqrt()).float()
    master = uni(-0.1, 0.1)
    master = torch.where(uni() < 0.25, sign() * torch.exp2(uni(-8, -1) * math.log2(10)), master)
    master = torch.where(uni() < 1 / 64, 0.0, master).float()
    if param_fp16:
        master = master.half().float()
    g = sign() * torch.exp2(uni(-9, math.log10(65504)) * math.log2(10))
    c = uni()
    g = torch.where(c < 1 / 8, 0.0, g)
    g = torch.where((c >= 1 / 8) & (c < 3 / 16), sign() * torch.randint(1, 1024, (n,), generator=gen, device=device) * 2.0 ** -24, g)
    g = torch.where((c >= 3 / 16) & (c < 1 / 4), sign() * 65504.0, g)
    if grad_dtype == torch.float32:
        g = torch.where((c >= 1 / 4) & (c < 5 / 16), sign() * torch.randint(1, 1 << 23, (n,), generator=gen, device=device) * 2.0 ** -149, g)
    g = g.to(grad_dtype)
    z = uni() < 1 / 32
    g, m, v = g.masked_fill(z, 0), m.masked_fill(z, 0), v.masked_fill(z, 0)
    return g, m, v, master
