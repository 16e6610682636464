"""The NGP optimizer tail (csrc/optimizer.cu) against float64 (tests/optimizer_ref.py), entry by entry, at the hash table's size:
- ngp_adam_ema with the EMA of lego_cfg (decay 0.95, betas 0.9 / 0.99, eps 1e-15) for fp16 / fp16, fp16 parameters with fp32 gradients
  and fp32 / fp32; at the lego and fox table sizes (the grid-stride loop wraps: asserted from the device's SM count), at n = 1, 2, 3, 5,
  6, 7 and 4099 (the scalar tail) and with n / 4 just below, at and just above the two unrolled slots of the largest grid; at steps 1, 2,
  3, 19 999, 20 000, 20 001, 30 000 and 40 000 (ExpDecay's boundaries; debias_old = debias_new = 1 by the last) with ExpDecay's learning
  rate, grad_scale 1, 1/2 and 1/3072.  m, v and master within adam_ema64's bound; param == rn16(master) (fp16) or master (fp32) bit
  for bit; the gradient zeroed or untouched; at step 1 master equals the Adam update within its bound (the old master drops out); a
  zero gradient with zero moments keeps master within a few u; every buffer's sentinel tail past n unchanged.
- ngp_train_sweep from hand-filled scratch, without a backward: fixed-point sums of every shape (zero, +-1, more than 24 significant
  bits, just inside the fp16 range, fp16 subnormals and rounding ties, one feature zero) at the lego and fox tables and at the sweep's
  own stride boundary.  The gradient it applied is fx_grad64(q) exactly -- ngp_adam_ema fed that fp16 gradient gives the same bits --
  and the state is within the bound; the scratch is cleared, and a second sweep on the same buffers, after new sums were added into the
  scratch, sees only those; sentinels past n_entries unchanged.  The weight slots: bwd_rows with bwd_ctas = 0, 1, 2, 3 (mod 4) and the
  SM count, slots past nparts NaN (so reading one shows); the sums the sweep formed (read back exactly through a sweep with beta1 = 0,
  where m1 = g) within gamma_nparts sum |terms| of the float64 sums, then Adam+EMA of the 3 072 + 7 168 weights within the bound.

Every bound is the worst case of optimizer_ref's error model, with no safety factor; a ratio is |kernel - float64| / bound.

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); every case prints its own line:
- ngp_adam_ema, all three dtype pairs: m and v 1.00 (printed to 3 digits; a result just above a power of two, rounded by almost half
  an ulp, meets u |x| with nothing to spare), master 0.75, master vs the Adam update at step 1 0.70, master kept under a zero gradient
  0.37 (of 8 u);
- ngp_train_sweep table, lego / fox / stride boundary: m 0.999, v 0.999, master 0.43 - 0.75; the applied gradient is fx_grad64(q) on every
  entry, the scratch is cleared and every sentinel kept;
- ngp_train_sweep weights: the slot sums 0.30 of gamma_nparts sum |terms| at 8 - 11 slots and 0.025 at 132; m 0.91, v 0.99, master 0.48;
- the file takes 31 s, 20 s of it in the five table cases."""
import math
import time

import numpy as np
import pytest
import torch

import optimizer_ref as O

pytestmark = pytest.mark.gpu

HYPER = dict(b1=0.9, b2=0.99, eps=1e-15, decay=0.95)
STEPS = [1, 2, 3, 19999, 20000, 20001, 30000, 40000]
GRAD_SCALES = [1.0, 0.5, 1.0 / 3072]
DTYPES = {"f16-f16": (torch.float16, torch.float16), "f16-f32": (torch.float16, torch.float32), "f32-f32": (torch.float32, torch.float32)}
PAD = 37                                        # sentinel elements past the end of every buffer
SENTINEL = -3.75
FX_SENTINEL = 0x5EED5EED5EED
WD_N, W_PART = 3072, 3072 + 7168


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _padded(x, fill=SENTINEL, pad=PAD):
    x = x.reshape(-1)
    buf = torch.full((x.numel() + pad,), fill, dtype=x.dtype, device="cuda")
    buf[:x.numel()] = x
    return buf


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _tail_ok(buf, n, fill=SENTINEL):
    return torch.equal(_bits(buf[n:]), _bits(torch.full_like(buf[n:], fill)))


class Tally:
    """Worst ratio per quantity and a description (with the kernel's inputs) of the first failing entry of each check."""

    def __init__(self):
        self.worst, self.fails = {}, []

    def bound(self, name, got, exact, err, tag, inputs):
        r = O.ratio(got.double(), exact, err)
        w = float(r.max()) if r.numel() else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), w)
        if not w <= 1:
            i = int(torch.argmax(torch.nan_to_num(r, nan=math.inf)))
            ins = ", ".join(f"{k} {float(v.reshape(-1)[i])!r}" for k, v in inputs.items())
            self.fails.append(f"{tag}{name}: {int((~(r <= 1)).sum())} entries outside the bound, first at {i}: got {float(got[i])!r}, "
                              f"float64 {float(exact[i])!r}, bound {float(err[i])!r} (err/bound {float(r[i]):.3g}); inputs {ins}")

    def exact(self, name, ok, tag):
        if not bool(ok):
            self.fails.append(f"{tag}{name}")

    def report(self):
        return ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items()))


def _adam(n, param, grad, m, v, master, h, zero_grad):
    from jnerf_b200 import lib, ops
    lib.call("ngp_adam_ema", ops._stream(), n, ops._p(param), ops._dt(param), ops._p(grad), ops._dt(grad), h.grad_scale, ops._p(m), ops._p(v),
             ops._p(master), h.lr, h.b1, h.b2, h.eps, h.step, h.decay, int(zero_grad))


def _sweep(n_entries, tab, fx, part, bwd_rows, wd, wr, h):
    """tab, wd, wr = (param, m, v, master)"""
    from jnerf_b200 import lib, ops
    p = ops._p
    lib.call("ngp_train_sweep", ops._stream(), n_entries, *map(p, tab), p(fx), p(part), int(bwd_rows), *map(p, wd), *map(p, wr), h.lr, h.b1, h.b2,
             h.eps, h.step, h.decay)


def _check_state(tally, tag, n, out, ref, inputs, pdt):
    """m, v, master of one call within adam_ema64's bound, param the rounding of master, everything finite"""
    param, m, v, master = (t[:n] for t in out)
    for name, got, k in (("m", m, 0), ("v", v, 2), ("master", master, 4)):
        tally.bound(name, got, ref[k], ref[k + 1], tag, inputs)
    tally.exact("everything finite", all(bool(torch.isfinite(t.float()).all()) for t in (param, m, v, master)), tag)
    expect = master.half() if pdt == torch.float16 else master
    tally.exact("param == rn(master)", torch.equal(_bits(param), _bits(expect)), tag)


# ------------------------------------------------------------------------------------------------------------ ngp_adam_ema
def _adam_sizes():
    """name -> n: the two table sizes (asserted to wrap the grid-stride loop), the scalar tail, and n / 4 just below, at and just above
    the 2 T float4 chunks one pass of the largest grid covers (T = 32 SMs x 256 threads, two unrolled slots)"""
    from jnerf_b200 import ops
    T = 32 * _sms() * 256
    sizes = {"lego": ops.HashLevels(1, log2_hashmap_size=19).n_params, "fox": ops.HashLevels(4, log2_hashmap_size=19).n_params}
    for name, n in sizes.items():
        blocks = min((-(-n // 4) + 511) // 512, 32 * _sms())
        assert blocks * 256 == T and n // 4 > 2 * T, f"the {name} table ({n} parameters) must wrap the grid-stride loop"
    sizes.update({str(n): n for n in (1, 2, 3, 5, 6, 7, 4099)})
    sizes.update({"2T-1": 4 * (2 * T - 1) + 3, "2T": 4 * 2 * T, "2T+1": 4 * (2 * T + 1) + 1})
    return sizes


@pytest.mark.parametrize("dt", list(DTYPES))
def test_adam_ema_against_fp64(dt):
    t0 = time.time()
    pdt, gdt = DTYPES[dt]
    tally = Tally()
    n_zero_grad = 0
    for si, (size, n) in enumerate(_adam_sizes().items()):
        g0, m0, v0, s0 = O.make_state(n, pdt == torch.float16, gdt, seed=1000 * si + len(dt) + (gdt == torch.float32), device="cuda")
        inputs = dict(g=g0, m=m0, v=v0, master=s0)
        g64, m64, v64, s64 = (x.double() for x in (g0, m0, v0, s0))
        triple = (g0 == 0) & (m0 == 0) & (v0 == 0)
        for k, step in enumerate(STEPS):
            h = O.Hyper(O.expdecay_lr(step), step, grad_scale=GRAD_SCALES[(k + si) % 3], **HYPER)
            zero_grad = (k + si) % 2
            tag = f"{dt} n={n} ({size}) {h} zero_grad={zero_grad}: "
            param, grad, m, v, master = (_padded(x) for x in (s0.to(pdt), g0, m0, v0, s0))
            _adam(n, param, grad, m, v, master, h, zero_grad)
            torch.cuda.synchronize()
            ref = O.adam_ema64(g64, m64, v64, s64, h, full=True)
            _check_state(tally, tag, n, (param, m, v, master), ref, inputs, pdt)
            if zero_grad:
                tally.exact("gradient zeroed", not bool(_bits(grad[:n]).any()), tag)
                n_zero_grad += 1
            else:
                tally.exact("gradient untouched", torch.equal(_bits(grad[:n]), _bits(g0)), tag)
            for name, buf in (("param", param), ("grad", grad), ("m", m), ("v", v), ("master", master)):
                tally.exact(f"{name} sentinel tail", _tail_ok(buf, n), tag)
            ms = master[:n].double()
            if step == 1:
                # debias_old = 0: the old master drops out and master is the Adam update, to the EMA's own roundings
                P, eP = ref[6], ref[7]
                tally.bound("step 1: master vs Adam p", ms, P, eP + 4 * O.U * abs(P) + 2 * O.TINY, tag, inputs)
            if bool(triple.any()):
                # zero gradient and moments: p = master, and (1 - d) + d debias_old = 1 - d^step = 1 / debias_new
                tally.bound("zero gradient: master kept", ms[triple], s64[triple], 8 * O.U * abs(s64[triple]) + 4 * O.TINY, tag,
                            {k_: t[triple] for k_, t in inputs.items()})
            del param, grad, m, v, master, ref, ms
    print(f"[optimizer-fp64] adam_ema {dt}: worst err/bound {tally.report()} ({time.time() - t0:.1f} s)")
    assert n_zero_grad > 0
    assert not tally.fails, "\n".join(tally.fails[:12])


# ------------------------------------------------------------------------------------------------------------ ngp_train_sweep
def _bwd_ctas(rows):
    return min(((rows + 127) // 128 + 1) // 2, _sms())


def _weights(seed):
    """(param, m, v, master) of both weight vectors, padded: the density weights' buffers and the colour weights'"""
    _, m, v, s = O.make_state(W_PART, True, torch.float16, seed=seed, device="cuda")
    return [tuple(_padded(x[lo:hi]) for x in (s.half(), m, v, s)) for lo, hi in ((0, WD_N), (WD_N, W_PART))]


def _clone(bufs):
    return tuple(b.clone() for b in bufs)


def _table_sizes():
    from jnerf_b200 import ops
    stride = 4 * 32 * _sms() * 256                              # entries one pass of the largest table grid covers (4 unrolled slots)
    sizes = {"lego": ops.HashLevels(1, log2_hashmap_size=19).n_entries, "fox": ops.HashLevels(4, log2_hashmap_size=19).n_entries}
    for name, n in sizes.items():
        assert min((n + 1023) // 1024, 32 * _sms()) * 256 * 4 == stride and n > stride, f"the {name} table must wrap the sweep's loop"
    sizes.update({"stride-1": stride - 1, "stride": stride, "stride+1": stride + 1})
    return sizes


@pytest.mark.parametrize("which,step", [("lego", 1), ("fox", 20000), ("stride-1", 2), ("stride", 30000), ("stride+1", 40000)])
def test_train_sweep_table_against_fp64(which, step):
    t0 = time.time()
    n = _table_sizes()[which]
    rng = np.random.default_rng(step + n)
    tally = Tally()
    _, m0, v0, s0 = O.make_state(2 * n, True, torch.float16, seed=n, device="cuda")
    tab = (_padded(s0.half(), pad=2 * PAD), _padded(m0, pad=2 * PAD), _padded(v0, pad=2 * PAD), _padded(s0, pad=2 * PAD))
    fx = _padded(torch.zeros(2 * n, dtype=torch.int64, device="cuda"), FX_SENTINEL, 2 * PAD)
    wd, wr = _weights(seed=n + 1)
    part = (torch.rand(_sms() * W_PART, device="cuda") - 0.5) * 1e-2
    for k in range(2):                                           # steps `step` and `step + 1` on the same buffers
        q = O.fx_sums(n, rng)
        if k == 1:
            q[rng.random(n) < 0.5] = 0                           # half the entries untouched by the second backward
        fx[:2 * n] += torch.from_numpy(q.reshape(-1)).cuda()     # added, as the backward adds: a sum left by the first sweep would show
        gq = torch.from_numpy(O.fx_grad64(q).reshape(-1)).cuda()
        h = O.Hyper(O.expdecay_lr(step + k), step + k, **HYPER)
        tag = f"{which} (n_entries={n}) {h}: "
        before = _clone(tab)
        _sweep(n, tab, fx, part, 1 << 18, wd, wr, h)
        # the same state through ngp_adam_ema with the fp16 gradient fx_grad64(q): the same bits iff the sweep applied exactly that
        replay = _clone(before)
        _adam(2 * n, replay[0], _padded(gq.half(), 0.0, 2 * PAD), *replay[1:], h, zero_grad=False)
        torch.cuda.synchronize()
        for name, a, b in zip(("param", "m", "v", "master"), tab, replay):
            tally.exact(f"step {k + 1}: {name} == ngp_adam_ema with fx_grad64(q)", torch.equal(_bits(a), _bits(b)), tag)
        ref = O.adam_ema64(gq, *(x[:2 * n].double() for x in before[1:]), h)
        inputs = dict(q=torch.from_numpy(q.reshape(-1)), m=before[1][:2 * n], v=before[2][:2 * n], master=before[3][:2 * n])
        _check_state(tally, tag, 2 * n, tab, ref, inputs, torch.float16)
        tally.exact("scratch cleared", not bool(fx[:2 * n].any()), tag)
        tally.exact("scratch sentinel tail", _tail_ok(fx, 2 * n, FX_SENTINEL), tag)
        for name, buf in zip(("param", "m", "v", "master"), tab):
            tally.exact(f"{name} sentinel tail", _tail_ok(buf, 2 * n), tag)
        n_q = int(np.count_nonzero(q))
        del before, replay, ref
    print(f"[optimizer-fp64] train_sweep table {which} ({n} entries, {n_q} nonzero sums in the second sweep): worst err/bound "
          f"{tally.report()} ({time.time() - t0:.1f} s)")
    assert not tally.fails, "\n".join(tally.fails[:12])


@pytest.mark.parametrize("ctas", [8, 9, 10, 11, "sms"])
def test_train_sweep_weights_against_fp64(ctas):
    t0 = time.time()
    sms = _sms()
    rows = 1 << 18 if ctas == "sms" else 256 * ctas - 37          # the last 128-row tile partial
    nparts = _bwd_ctas(rows)
    assert nparts == (sms if ctas == "sms" else ctas) and nparts % 4 == (sms if ctas == "sms" else ctas) % 4
    gen = torch.Generator(device="cuda").manual_seed(nparts)
    part = torch.full(((sms + 2) * W_PART,), math.nan, device="cuda")         # slots at or past nparts: NaN, never read
    mag = torch.exp2(torch.empty(nparts * W_PART, device="cuda").uniform_(-20, 6, generator=gen))
    part[:nparts * W_PART] = torch.where(torch.rand(nparts * W_PART, device="cuda", generator=gen) < 0.5, -mag, mag)
    terms = part[:nparts * W_PART].view(nparts, W_PART).double()
    exact, mass = terms.sum(0), terms.abs().sum(0)
    n = 1000                                                      # a small table with zero sums
    tab0 = tuple(_padded(x) for x in (torch.zeros(2 * n, dtype=torch.float16, device="cuda"),) + (torch.zeros(2 * n, device="cuda"),) * 3)
    fx = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
    w0 = _weights(seed=nparts)
    tally = Tally()
    step = STEPS[nparts % len(STEPS)]
    # beta1 = 0: m1 = fma(0, m, fl(1 g)) = g, the sum the sweep formed, exactly
    wd, wr = _clone(w0[0]), _clone(w0[1])
    _sweep(n, _clone(tab0), fx, part, rows, wd, wr, O.Hyper(0.1, step, b1=0.0, b2=0.99, eps=1e-15, decay=0.95))
    torch.cuda.synchronize()
    g = torch.cat([wd[1][:WD_N], wr[1][:W_PART - WD_N]])
    gamma = nparts * O.U / (1 - nparts * O.U)
    tally.bound("weight-gradient sum", g, exact, gamma * mass + O.TINY, f"nparts={nparts}: ", dict(sum_abs=mass))
    # the real hyper-parameters on the same state, from the gradient the sweep formed
    h = O.Hyper(O.expdecay_lr(step), step, **HYPER)
    wd, wr = _clone(w0[0]), _clone(w0[1])
    _sweep(n, _clone(tab0), fx, part, rows, wd, wr, h)
    torch.cuda.synchronize()
    for name, (lo, hi), before, after in (("density", (0, WD_N), w0[0], wd), ("colour", (WD_N, W_PART), w0[1], wr)):
        nn_ = hi - lo
        tag = f"{name} weights, nparts={nparts}, {h}: "
        ref = O.adam_ema64(g[lo:hi].double(), *(x[:nn_].double() for x in before[1:]), h)
        _check_state(tally, tag, nn_, after, ref, dict(g=g[lo:hi], m=before[1], v=before[2], master=before[3]), torch.float16)
        for bname, buf in zip(("param", "m", "v", "master"), after):
            tally.exact(f"{bname} sentinel tail", _tail_ok(buf, nn_), tag)
    print(f"[optimizer-fp64] train_sweep weights, bwd_rows {rows} -> {nparts} slots: worst err/bound {tally.report()} "
          f"({time.time() - t0:.1f} s)")
    assert not tally.fails, "\n".join(tally.fails[:12])
