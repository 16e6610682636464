"""CPU checks of the restatements and bounds that test_gpu_march_reference.py and test_gpu_grid_update_reference.py rely on (march_ref).

const_dt closed form (march_count_kernel's stage1): wherever the shortcut is taken it gives the 32 lane values and the next chunk's start
of the sequential float additions, bit for bit, in every binade 117..140 -- random starts, the last 32 floats below each power of two,
and the one binade (e0 = 117, t in [2^-10, 2^-9)) where h / ulp is a tie.  Dropping the e1 test takes chunks across a power of two and
fails.  With the production step h = fl(sqrt(3)/1024)/2 the e1 test is what carries the guard: a 32-step chunk (0.027) does not fit in
any binade below 122, the tie binade included, and from 141 up fl(t + h) = t in every lane.  So dropping the tie test, or widening the
window to 116 or 141, changes no sample for this h; the tie test is still needed for a shorter step, which the family of steps below
shows (a tie binade wide enough to hold a chunk), and the window is shown to be conservative rather than load-bearing.

Mean: the float32 emulation of mean_partial_kernel / mean_final_kernel stays inside gamma(47) * mean on adversarial grids, and reaches
at least a tenth of it (a bound 10x coarser, e.g. the 1e-5 relative of test_gpu_ops.py, would fail that); summing a block serially in
one thread, i.e. the reduction reordered without adjusting the bound, leaves it."""
import numpy as np
import pytest

import march_ref as M

SHORT_H = np.float32(1001 * 2.0 ** -34)      # a step with h / ulp = 500.5 in binade 117 and a chunk (1.9e-6) far inside one binade


def _starts(seed=0, per_binade=3000):
    rng = np.random.default_rng(seed)
    parts, tags = [], []
    for e in range(117, 141):
        m = rng.integers(0, 1 << 23, per_binade).astype(np.uint32)
        parts.append(((np.uint32(e) << 23) | m).view(np.float32))
        top = np.float32(2.0 ** (e - 126))                                     # 2^(e-127+1): the next power of two
        parts.append((top.view(np.uint32) - np.arange(1, 33, dtype=np.uint32)).view(np.float32))
        tags += [e] * (per_binade + 32)
    return np.concatenate(parts), np.array(tags)


def test_closed_form_is_the_sequential_additions():
    tc, e = _starts()
    bad, taken = M.closed_form_mismatches(tc)
    assert not bad.any()
    # the shortcut really runs (binades wide enough to hold a chunk) and really declines (chunks across a power of two, narrow binades)
    assert taken.sum() > 0.5 * tc.size and (~taken).sum() > 1000
    assert not taken[e < 122].any() and taken[e >= 122].any()
    # the tie binade: h / ulp = x.5 there and only there
    r = M.H_CONST * np.float32(2.0 ** (150 - 117))
    assert r - np.floor(r) == 0.5
    assert all(M.H_CONST * np.float32(2.0 ** (150 - k)) % 1 != 0.5 for k in range(118, 141))


def test_e1_mutant_fails():
    tc, e = _starts()
    bad, _ = M.closed_form_mismatches(tc, mutant="no_e1")
    assert bad.sum() > 1000
    assert bad[np.isin(np.arange(tc.size) % 3032, np.arange(3000, 3032))].any()     # among the last floats below a power of two


def test_tie_mutant_fails_for_a_step_that_fits_its_binade():
    rng = np.random.default_rng(3)
    tc = ((np.uint32(117) << 23) | rng.integers(0, 1 << 23, 4000).astype(np.uint32)).view(np.float32)
    bad, taken = M.closed_form_mismatches(tc, SHORT_H)
    assert not bad.any() and not taken.any()                                  # the tie test declines every start
    bad, _ = M.closed_form_mismatches(tc, SHORT_H, mutant="no_tie")
    assert bad.sum() > 1000                                                  # round-to-even alternates q: t_k != t_0 + k q


@pytest.mark.parametrize("mutant", ["no_tie", "window_116", "window_141"])
def test_guards_implied_by_e1_for_the_production_step(mutant):
    """For h = fl(sqrt(3)/1024)/2 these guards change nothing: binades 116 and 117 are narrower than a chunk (the e1 test declines),
    and at 141 q = 0 and fl(t + h) = t, so the shortcut equals the additions."""
    tc, _ = _starts()
    extra = [((np.uint32(e) << 23) | np.arange(0, 1 << 23, 4099, dtype=np.uint32)).view(np.float32) for e in (116, 141, 142)]
    tc = np.concatenate([tc] + extra)
    bad, _ = M.closed_form_mismatches(tc, mutant=mutant)
    assert not bad.any()
    e141 = extra[1]
    assert ((e141 + M.H_CONST) == e141).all()


def _adversarial_grids():
    rng = np.random.default_rng(1)
    yield "uniform", (rng.random(M.G3) * 0.02).astype(np.float32)
    for v in (0.0051, 0.0099, 0.011, 1.0 / 3.0):
        yield f"const {v}", np.full(M.G3, np.float32(v), np.float32)
    g = np.where(rng.random(M.G3) < 0.1, np.float32(0.05), np.float32(-1)).astype(np.float32)
    yield "sparse, untrained cells", g


def test_mean_bound_holds_and_is_tight():
    worst = 0.0
    for name, g in _adversarial_grids():
        s, _ = M.mean_f64(g)
        err = abs(float(M.mean_f32(g)) - s)
        b = M.mean_bound(g)
        assert err <= b, name
        worst = max(worst, err / b)
    print(f"[mean-cpu] worst err / bound {worst:.3f}")
    assert worst >= 0.1                                                      # a bound 10x coarser would not notice a wrong order


def test_mean_mutants_fail():
    coarse_worst, reordered_out = 0.0, 0
    for name, g in _adversarial_grids():
        s, _ = M.mean_f64(g)
        coarse_worst = max(coarse_worst, abs(float(M.mean_f32(g)) - s) / (M.gamma(47 * 10) * s))
        reordered_out += abs(float(M.mean_f32(g, serial=8192)) - s) > M.mean_bound(g)
    assert coarse_worst < 0.1                                                # the coarser bound fails the tightness check above
    assert reordered_out >= 3                                                # one serial thread per block leaves the bound


def test_splat_bound_entries():
    x = np.array([0.0, -0.0, 1.0, -1.0, 10.0, -83.0, -90.0, -104.0, 65504.0, -65504.0, np.inf, -np.inf])
    ref, b = M.splat_ref(x)
    assert ref[0] == M.THICK and b[0] < 6 * M.U * M.THICK              # 2 ulp of exp(0) = 4u, one rounding u
    assert np.isinf(ref[8]) and np.isinf(ref[10]) and ref[9] == 0 and ref[11] == 0
    assert 0 < ref[5] < 2.0 ** -126 and ref[5] > b[5]                         # a subnormal product the bound still separates from 0
    assert ref[7] < 2.0 ** -150 and b[7] >= ref[7]                            # rounds to 0 within the bound
    assert M.ulp32(1.0) == 2.0 ** -23 and M.ulp32(1e-40) == 2.0 ** -149


def test_n_emit_reader_and_row_t():
    R = 5
    ws = np.zeros(8 * R + 1024, np.uint8)
    counts = np.arange(R, dtype=np.uint32) * 7
    ne = np.arange(R, dtype=np.uint32) + 60
    ws[:4 * R] = counts.view(np.uint8)
    ws[4 * R:8 * R] = ne.view(np.uint8)
    assert np.array_equal(M.n_emit(ws, R), ne)
    rng = np.random.default_rng(2)
    o = rng.uniform(-1, 2, (1000, 3)).astype(np.float32)
    d = rng.normal(size=(1000, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    t = rng.uniform(1e-3, 3, 1000).astype(np.float32)
    lo, hi = np.float32(-1.5), np.float32(2.5)
    p = (t[:, None].astype(np.float64) * d + o).astype(np.float32)                 # fma(t, d, o)
    rows = ((p - lo) / (hi - lo)).astype(np.float32)
    tr = M.row_t(rows, o, d, (lo, hi))
    assert np.abs(tr - t).max() <= 8 * np.sqrt(3) * 2.0 ** -23 * 4


def test_unknown_mutant_name_is_refused():
    with pytest.raises(AssertionError):
        M.closed_form(np.ones(4, np.float32), mutant="no-tie")


def test_step_and_chunk_helpers():
    rng = np.random.default_rng(4)
    t0 = (rng.random(50) * M.H_CONST).astype(np.float32)
    seq = M.sequential(t0, n=2048)
    assert np.array_equal(seq[:, :33], M.sequential(t0))
    cross = M.chunk_crosses_binade(seq)
    assert cross.shape == (50, 64) and cross.any(1).all() and not cross.all()
    ray = np.repeat(np.arange(50), 40)
    k_true = np.sort(rng.integers(0, 2048, (50, 40)), axis=1).ravel()
    t = seq[ray, k_true].astype(np.float64) * (1 + 1e-7 * rng.uniform(-1, 1, ray.size))   # what row_t's recovery leaves
    k, err = M.step_of_rows(t, ray, seq)
    assert np.array_equal(k, k_true) and err < M.H_CONST / 100


def test_index_wrap_of_grid_samples_is_harmless():
    """generate_samples_kernel forms ((i + step * n) * 56924617 + j * 19349663 + 96925573) % G3 in 32-bit arithmetic.  G3 = 2^21 divides
    2^32, so the wraps of step * n and of the products change no index: a 64-bit evaluation gives the same cells at every step."""
    for n in (M.G3, 3 * M.G3, M.G3 // 4, 3 * M.G3 // 4):
        for step in (1, -(-(1 << 32) // n), 2 ** 31 - 1):
            i = np.arange(0, n, 9973, dtype=np.uint64)
            for j in (0, 9):
                exact = ((i + np.uint64(step) * np.uint64(n)) * np.uint64(56924617) + np.uint64(j * 19349663 + 96925573)) % np.uint64(M.G3)
                w = (i + np.uint64(step) * np.uint64(n)) & np.uint64(0xFFFFFFFF)
                w = (w * np.uint64(56924617) + np.uint64(j * 19349663 + 96925573)) & np.uint64(0xFFFFFFFF)
                assert np.array_equal(exact, w % np.uint64(M.G3))
            assert step * n >= 1 << 32 or step == 1
