"""Rehearsal of the bound of test_gpu_optimizer_reference.py on the CPU (optimizer_ref has the bound and the fp32 emulation).

Not too tight: a numpy float32 emulation of adam_one, operation for operation, lies inside adam_ema64's bound on every entry of m, v and
master, at the steps, learning rates, grad_scale values and input distributions the GPU test uses.

Not too loose: on the same inputs each mutant of adam_one's arithmetic puts entries outside the bound -- debias_old not applied at step 1
(the old master kept), 1 - decay swapped with decay, lr in place of step_size, b1 and b2 swapped, eps inside the square root,
grad_scale applied twice and the EMA reading the updated p instead of the old master.  The fixed-point gradient is exact:
fx_grad64 agrees with a float64 -> float32 -> float16 rounding of Python's exact integers and with rounding ties resolved to even."""
import numpy as np
import pytest
import torch

import optimizer_ref as O

N = 1 << 15
STEPS = [1, 2, 3, 19999, 20000, 20001, 30000, 40000]
GRAD_SCALES = [1.0, 0.5, 1.0 / 3072]
DTYPES = {"f16-f16": (True, torch.float16), "f16-f32": (True, torch.float32), "f32-f32": (False, torch.float32)}


def _cases():
    for dt, (p16, gdt) in DTYPES.items():
        g, m, v, ms = (t.numpy() for t in O.make_state(N, p16, gdt, seed=len(dt) + int(p16) * 7 + (gdt == torch.float32)))
        for k, step in enumerate(STEPS):
            yield dt, O.Hyper(O.expdecay_lr(step), step, grad_scale=GRAD_SCALES[k % 3]), (g.astype(np.float32), m, v, ms)


def _out_of_bound(h, inp, mutant=None):
    g, m, v, ms = inp
    m1, v1, s1 = O.adam_one_f32(g, m, v, ms, h, mutant)
    ref = O.adam_ema64(*(x.astype(np.float64) for x in (g, m, v, ms)), h)
    r = [O.ratio(got.astype(np.float64), ref[2 * j], ref[2 * j + 1]) for j, got in enumerate((m1, v1, s1))]
    return r


def test_bound_holds_for_the_fp32_emulation():
    worst = {}
    for dt, h, inp in _cases():
        for name, r in zip(("m", "v", "master"), _out_of_bound(h, inp)):
            assert (r <= 1).all(), f"{dt} {h}: {name} outside the bound at {np.argwhere(r > 1)[:4].ravel().tolist()}"
            worst[f"{name} {dt}"] = max(worst.get(f"{name} {dt}", 0.0), float(r.max()))
        m1, v1, s1 = O.adam_one_f32(*inp, h)
        assert np.isfinite(m1).all() and np.isfinite(v1).all() and np.isfinite(s1).all()
    print("[optimizer-cpu] fp32 emulation, worst err/bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


def test_late_steps_debias_to_one():
    h = O.Hyper(0.1, 40000)
    assert h.debias_old == 1.0 and h.debias_new == 1.0 and h.step_size == h.lr
    h1 = O.Hyper(0.1, 1)
    assert h1.debias_old == 0.0 and h1.debias_new == 1.0 / (1.0 - h1.decay) and h1.step_size == h1.lr * np.sqrt(1 - h1.b2) / (1 - h1.b1)


@pytest.mark.parametrize("mutant", O.MUTANTS)
def test_mutant_fails_the_bound(mutant):
    out, total = {}, 0
    for dt, h, inp in _cases():
        n_out = sum(int((r > 1).sum()) for r in _out_of_bound(h, inp, mutant))
        if n_out:
            out[f"{dt}/step {h.step}"] = n_out
        total += n_out
    print(f"[optimizer-cpu] mutant {mutant}: {total} entries outside the bound in {len(out)} of {3 * len(STEPS)} cases {sorted(out)[:4]}")
    assert total > 0


def _round_int(x, s):
    """x rounded to a multiple of 2^s, ties to even"""
    if s <= 0:
        return x
    q, r = divmod(abs(x), 1 << s)
    if r > 1 << (s - 1) or (r == 1 << (s - 1) and q & 1):
        q += 1
    return (q << s) * (1 if x >= 0 else -1)


def test_fx_grad64_is_the_double_rounding():
    rng = np.random.default_rng(0)
    q = O.fx_sums(1 << 16, rng)
    h = O.fx_grad64(q)
    kinds = {"zero": q == 0, "one": np.abs(q) == 1, "subnormal": (q != 0) & (np.abs(q) < 1 << 18), "near 65504": np.abs(q) > 65000 << 32,
             "rounds in fp32": (np.abs(q) > 1 << 24) & (q.astype(np.float32).astype(np.int64) != q)}
    for name, k in kinds.items():
        assert k.sum() > 100, name
    assert ((q[:, 0] == 0) != (q[:, 1] == 0)).sum() > 1000                       # one feature zero, the other not
    # the same two roundings in Python's exact integers: 24 significant bits, then 11 (or the subnormal quantum of 2^8 units)
    exact = []
    for x in (int(x) for x in q.ravel()[:20000]):
        y = _round_int(x, max(abs(x).bit_length() - 24, 0))
        exact.append(_round_int(y, max(abs(y).bit_length() - 11, 8)) * 2.0 ** -32)
    assert np.array_equal(h.ravel()[:20000], np.array(exact))
    # ties in the subnormal range go to even: (2k + 1) 2^7 units is half way between k and k + 1 subnormal steps of 2^8 units
    k = np.arange(0, 512, dtype=np.int64)
    tie = O.fx_grad64(np.stack([(2 * k + 1) * 128, -(2 * k + 1) * 128], 1))
    even = (k + (k & 1)) * 2.0 ** -24
    assert np.array_equal(tie[:, 0], even) and np.array_equal(tie[:, 1], -even)
    assert O.fx_grad64(np.array([[65504 << 32, 0]]))[0, 0] == 65504.0
