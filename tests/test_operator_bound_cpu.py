"""Rehearsal of the bounds of test_gpu_operator_reference.py on the CPU (operator_ref has the bounds and the models).

Not too tight: host evaluations of the same operations must lie inside every bound -- the oracle's serial fp32 and fp16 hash-grid scatters
(one product and one add per row: the bound with runs of one row, R_e = cnt_e), a numpy model of the backward's run partition summed in
fp32 and fp16 in two random orders, the oracle's fp32 and fp32-accumulated fp16 forwards, the fp32 SH and a numpy MLP that accumulates
in fp32.  The forward model must also reproduce the oracle bit for bit, which pins Geometry's cells and weights to the kernel's.

Not too loose: on the same inputs each mutant of the kernels' arithmetic must put entries outside its bound -- swapped halves of a paired
x-neighbour reduction, the last run of each chunk dropped, stale corner indices when only gz changes, fp16 subnormal run sums flushed to
zero, corner weights c and c ^ 1 swapped in the forward, a hidden layer's ReLU mask skipped in the backward and the rows of a partial last
tile left out of the weight gradients.

Inputs: ray-ordered samples of the oracle's march (1024 rays through a spherical shell, compacted to 2^15 rows) with a fifth of
them snapped to cell faces, 0 or 1; training-like output gradients (operator_ref.training_dy)."""
import functools

import numpy as np
import pytest
import torch

import oracle_lib as ol
from ngp_fwd_ref import fma32, sh_f32, sh_f64, sh_interval
from operator_ref import (DEFAULT_PRIMES, L, RUN, Geometry, check_bwd, check_fwd, check_mlp, face_values, hash_bwd_bound, hash_fwd_f64,
                          level_scales, host_scales, mlp_probe_weights, mlp_weights, model_hash_bwd, model_mlp, reductions, sh_special_directions,
                          snap_rows, training_dy)

N_ROWS = 1 << 15
TABLES = {"aabb1-T14": (1, 14, DEFAULT_PRIMES), "aabb4-T19": (4, 19, DEFAULT_PRIMES), "primes-T14": (1, 14, (3, 2654435761, 805459861))}
BWD_MUTANTS = ["swap-halves", "drop-last-run", "stale-gz", "ftz"]


@functools.lru_cache(None)
def _samples():
    o, d = ol.random_rays(1024, seed=3)
    bits = ol.sphere_bitfield(0.3, shell=0.03)[0]
    coords, _, ns, _ = ol.march(o, d, bits, max_samples=1 << 20)
    cc, _, cnt = ol.compact(coords, ns, N_ROWS)
    n = min(int(cnt[0]), N_ROWS)
    assert n == N_ROWS, n
    return cc[:n]


@functools.lru_cache(None)
def _case(table):
    aabb, log2T, primes = TABLES[table]
    cfg = ol.HashCfg(aabb, log2_hashmap_size=log2T)
    scales = host_scales(cfg)
    rng = np.random.default_rng(log2T + aabb)
    x = snap_rows(_samples()[:, :3].copy(), face_values(scales, range(0, L, 3), rng), rng, share=0.2)
    return cfg, scales, primes, Geometry(cfg, x, scales, primes), x


def _fwd_chain(geo, grid, swap=False):
    """the kernel's forward in numpy: an fmaf chain over the corners per feature (swap: weights of corners c and c ^ 1 exchanged)"""
    g2 = np.asarray(grid).reshape(-1, 2).astype(np.float32)
    out = np.zeros((geo.n, 2 * L), np.float32)
    for l in range(L):
        a = np.zeros((geo.n, 2), np.float32)
        for c in range(8):
            a = fma32(geo.w[l, :, c ^ 1 if swap else c][:, None], g2[geo.idx[:, l, c]], a)
        out[:, 2 * l:2 * l + 2] = a
    return out


def test_runs_are_long_at_the_coarse_levels():
    """the inputs give the run reuse something to do: dozens of rows per run would need more than RUN rows; at least several"""
    cfg, scales, primes, geo, x = _case("aabb1-T14")
    dy = training_dy(geo.n, np.random.default_rng(0), True)
    R, mean_run = reductions(geo, dy)
    print(f"[operator-cpu] RUN {RUN}: mean rows per run by level {np.round(mean_run, 2).tolist()}")
    assert mean_run[0] > 4 and mean_run[-1] < mean_run[0]


@pytest.mark.parametrize("table", list(TABLES))
def test_hash_fwd_bound_and_mutant(table):
    cfg, scales, primes, geo, x = _case(table)
    rng = np.random.default_rng(1)
    for dt in (np.float32, np.float16):
        grid = (rng.uniform(-1, 1, cfg.n_params) * (1e-4 if dt == np.float16 else 1.0)).astype(dt)
        y, e = hash_fwd_f64(geo, grid)
        with level_scales(scales, primes):
            ref = ol.hash_fwd(cfg, x, grid, acc32=True)
        ok, ratio = check_fwd(ref, y, e)
        assert ok.all(), f"{dt.__name__}: the oracle's forward is outside the bound at {np.argwhere(~ok)[:4].tolist()}"
        chain = _fwd_chain(geo, grid)
        if dt == np.float16:
            chain = chain.astype(np.float16)
        assert np.array_equal(chain.view(np.uint16 if dt == np.float16 else np.uint32), ref.view(np.uint16 if dt == np.float16 else np.uint32)), \
            "the numpy fmaf chain differs from the oracle: Geometry's weights or cells are not the kernel's"
        mut = _fwd_chain(geo, grid, swap=True)
        mok, _ = check_fwd(mut.astype(dt), y, e)
        print(f"[operator-cpu] fwd {table}/{dt.__name__}: worst ratio {ratio.max():.3g}; swapped corner weights: {int((~mok).sum())} entries out")
        assert (~mok).sum() > 0.1 * mok.size


@pytest.mark.parametrize("table", list(TABLES))
def test_hash_bwd_bound_holds_for_host_scatters(table):
    cfg, scales, primes, geo, x = _case(table)
    for fp16 in (False, True):
        dy = training_dy(geo.n, np.random.default_rng(2), fp16)
        with level_scales(scales, primes):
            g, a, cnt = ol.hash_bwd_f64(cfg, x, dy.astype(np.float32))
            serial = ol.hash_bwd(cfg, x, dy)
        R, _ = reductions(geo, dy)
        stats = []
        # the serial oracle: runs of one row, every contribution its own reduction
        bound = hash_bwd_bound(a, cnt.astype(np.int64), fp16, run=1)
        err = np.abs(serial.astype(np.float64) - g)
        assert (err <= bound).all(), f"serial oracle: {int((err > bound).sum())} entries outside the bound"
        assert (serial[cnt == 0] == 0).all()
        for seed in range(2):
            got = model_hash_bwd(geo, dy, fp16, np.random.default_rng(seed))
            n_out, n_untouched, worst, tight = check_bwd(got, g, a, cnt, R, fp16)
            stats.append(worst)
            assert n_out == 0 and n_untouched == 0, (seed, n_out, n_untouched)
        print(f"[operator-cpu] bwd {table}/{'fp16' if fp16 else 'fp32'}: worst ratio over 2 orders {max(stats):.3g}; "
              f"touched entries with a bound below 1 % of A_e: {tight:.3f}")
        if fp16:
            assert tight > 0.2        # the rest are entries of a few subnormal terms, where 2^-25 per rounding dominates


@pytest.mark.parametrize("mutant", BWD_MUTANTS)
@pytest.mark.parametrize("table", ["aabb1-T14", "aabb4-T19"])
def test_hash_bwd_mutants_fail(table, mutant):
    cfg, scales, primes, geo, x = _case(table)
    dy = training_dy(geo.n, np.random.default_rng(2), True)
    with level_scales(scales, primes):
        g, a, cnt = ol.hash_bwd_f64(cfg, x, dy.astype(np.float32))
    R, _ = reductions(geo, dy)
    got = model_hash_bwd(geo, dy, True, np.random.default_rng(0), mutant=mutant)
    n_out, n_untouched, worst, _ = check_bwd(got, g, a, cnt, R, True)
    print(f"[operator-cpu] mutant {mutant} on {table}: {n_out} entries outside the bound, {n_untouched} untouched entries written")
    assert n_out + n_untouched > 0


def test_sh_bound_and_contraction():
    rng = np.random.default_rng(4)
    d = np.concatenate([sh_special_directions(rng), _samples()[:20000, 4:]])
    lo, hi = (t.numpy() for t in sh_interval(d))
    for contract in (True, False):
        v = sh_f32(d, contract).astype(np.float16).astype(np.float64)
        assert ((v >= lo) & (v <= hi)).all(), contract
    ref = ol.sh(d, np.float32)
    assert np.array_equal(sh_f32(d, contract=False).view(np.uint32), ref.view(np.uint32))      # the oracle is the uncontracted form
    o = ol.sh(d, np.float32).astype(np.float64)
    v = sh_f64(d)[0].numpy()
    assert np.abs(o - v).max() < 1e-5


def _mlp_case(nhm, n, probe, seed=5):
    rng = np.random.default_rng(seed)
    W = mlp_probe_weights(nhm) if probe else mlp_weights(nhm, rng)
    X = np.clip(rng.standard_normal((n, 32)), -4, 4).astype(np.float16)
    nv = 16 if nhm == 0 else 3
    dY = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    dY[:, nv:] = 0
    return W, X, dY, nv


@pytest.mark.parametrize("probe", [False, True], ids=["realistic", "probe"])
@pytest.mark.parametrize("nhm", [0, 1, 2, 3])
def test_mlp_bound_holds_for_fp32_model(nhm, probe):
    for n in (1, 127, 129, 1000):
        W, X, dY, nv = _mlp_case(nhm, n, probe)
        inter, Y, temps, dX, dW = model_mlp(W, X, dY, nhm, nv)
        t = torch.from_numpy
        worst, fails = check_mlp(t(W), t(X), t(inter), t(Y), t(dY), t(temps), t(dX), t(dW), nhm, nv, n, 1)
        assert not fails, (n, fails)
        if probe:
            assert np.array_equal(Y[:, :16], X[:, :16]) and np.array_equal(dX[:, :16], np.where(X[:, :16] != 0, dY, 0).astype(np.float16))
    print(f"[operator-cpu] mlp nhm={nhm} {'probe' if probe else 'realistic'}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("mutant,nhm,n", [("skip-mask", 1, 1000), ("skip-mask", 3, 129), ("drop-tail-tile", 0, 129), ("drop-tail-tile", 2, 300),
                                          ("drop-tail-tile", 3, 127)])
def test_mlp_mutants_fail(mutant, nhm, n):
    W, X, dY, nv = _mlp_case(nhm, n, False)
    t = torch.from_numpy
    inter, Y, temps, dX, dW = model_mlp(W, X, dY, nhm, nv, mutant=mutant)
    _, fails = check_mlp(t(W), t(X), t(inter), t(Y), t(dY), t(temps), t(dX), t(dW), nhm, nv, n, 1)
    print(f"[operator-cpu] mutant {mutant} nhm={nhm} n={n}: {fails[:2]}")
    assert fails
