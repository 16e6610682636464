"""The per-operator NGP kernels -- ngp_hash_fwd / ngp_hash_bwd / ngp_sh_fwd (csrc/hash_encode.cu) and ngp_mlp_fwd / ngp_mlp_bwd /
ngp_mlp_bwd_dgrad (csrc/mlp_tc.cu) -- against float64 at training batch sizes, entry by entry (operator_ref has the references, the bounds
and their derivations; test_operator_bound_cpu.py rehearses them on host models and shows that mutants of the kernels fail them).

Inputs.  The ray-ordered rows of a training step: 8192 rays marched through a spherical shell and compacted at 2^18 rows (the march
fixture of test_gpu_network_fwd_reference.py), so that consecutive rows stay in one cell for several rows at the coarse levels and the
run-length reuse of the hash kernels is exercised.  "faces": the first 2^18 - 77 of them with a fifth of their 8-row blocks given a
coordinate on a cell face of levels 0, 3, ..., 15 (fmaf(x, scale, 0.5) an integer), at 0 or at 1.  "small": the first 0, 1, 15, 16, 17,
255, 256 and 257 rows (chunk and block edges of the RUN = 16-row partition).  Tables: aabb 1 at T = 2^14 and 2^19, aabb 4 at 2^19 (dense and
hashed levels), and T = 2^14 with another hash_func, p1 * 2654435761 ^ p0 * 3 ^ 805459861 * p2.

Hash-grid forward, fp32 and fp16 tables: the output equals the oracle's per-point evaluation bit for bit (orc_hash_fwd_f32; fp16:
orc_hash_fwd_f16_acc32) -- reusing a cell's corner values must not change a bit; a random permutation of the rows gives the same bits
back; the fp16 encoding equals the fused forward's saved enc; and every entry lies within gamma_8 sum_c |w_c v_c| of the exact sum (fp16:
is a rounding of a value within it).

Hash-grid backward, fp32 and fp16 gradients, on training-like dL/denc (magnitudes 1e-8 .. 1e-3, zero rows inside runs, one feature zero):
every entry within the bound of operator_ref built on R_e, the reductions of the kernel's own partition; an entry no row reaches holds 0.
Each case prints the mean rows per run at level 0, the zero rows skipped inside runs, the paired x-neighbour reductions, the share of
non-zero fp16 gradients that are subnormal and the share of touched entries whose bound is below 1 % of A_e.

SH, fp32 and fp16, 2^18 directions: the axes, the cube diagonals, components at 0, 0.5 and 1, directions where 1 - 5 z^2, 5 z^2 - 3,
x^2 - y^2, -3 x^2 + y^2 and -x^2 + 3 y^2 cancel, and the march's directions.  Every entry equals ngp_fwd_ref.sh_f32(contract=True) bit for
bit: sh_kernel's SASS (cuobjdump -sass, sm_90a, both instantiations) contracts the same seven terms as the fused kernels -- o[6] = fma(z2,
C6A, -C6B), o[8] = fma(x2, C8, -(y2 C8)), the inner differences of o[9] fma(x2, -3, y2), of o[11] and o[13] fma(z2, -5, 1), of o[12]
fma(z2, 5, -3) and of o[15] fma(y2, 3, -x2) -- with x = fma(d, 2, -1) and every other operation a separate multiply or add (o[14]'s x2 - y2
an FADD).  And every entry lies in the float64 interval of ngp_fwd_ref.sh_interval.

Fully-fused MLP, nhm = 0 .. 3 hidden matmuls at n = 1, 127, 129, 2^18 - 77 and 2^18 rows (at 2^18 each forward CTA takes 3-4 tiles and
each backward CTA 8-16), with realistic weights and with the exact probe weights of operator_ref.mlp_probe_weights: every stored inter
block, Y, temps block and dX is checked layer by layer from the kernel's own operands; dW within the accumulation bound; padded output
rows of dW exactly 0; ngp_mlp_bwd_dgrad with the feature-major (16, n) dY equals ngp_mlp_bwd's temps and dX bit for bit.

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bound over all cases:
- hash forward: 0.64 (fp32), 0.30 (fp16); every case equal to the oracle bit for bit, permutation-invariant and equal to the fused enc;
- hash backward: 0.29 (fp32), 0.59 (fp16).  On the 2^18-row sets level 0 averages 7.0-9.4 rows per run, 0.17-0.36 M zero rows are skipped
  inside runs, 0.09-3.8 M reductions are paired, 18-84 % of the non-zero fp16 gradients are subnormal, and the fp16 bound is below 1 % of
  A_e on 6-34 % of the touched entries (the T = 2^14 tables, whose entries collect the most runs, lowest); the fp32 bound on all of them;
- SH: every feature equal to sh_f32 and inside its interval, fp32 and fp16;
- MLP, realistic weights: inter 0.026, Y 0.014, temps 0.045, dX 0.017, dW 0.021; probe weights: 0 for every stored block, dW 0.014.
The whole file ran in 118 s, most of it the host-side oracle and numpy geometry at 2^18 rows x 16 levels."""
import functools
import time

import numpy as np
import pytest
import torch

import oracle_lib as ol
from ngp_fwd_ref import sh_f32, sh_f64, sh_interval
from operator_ref import (DEFAULT_PRIMES, L, Geometry, check_bwd, check_fwd, check_mlp, device_scales, face_values, hash_fwd_f64,
                          level_scales, mlp_bwd_ctas, mlp_probe_weights, mlp_weights, partition, reductions, sh_special_directions, snap_rows,
                          training_dy)

pytestmark = pytest.mark.gpu

N = 1 << 18
SMALL = [0, 1, 15, 16, 17, 255, 256, 257]
TABLES = {"aabb1-T14": (1, 14, DEFAULT_PRIMES), "aabb1-T19": (1, 19, DEFAULT_PRIMES), "aabb4-T19": (4, 19, DEFAULT_PRIMES),
          "primes-T14": (1, 14, (3, 2654435761, 805459861))}
_LEVELS = {}


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _levels(table):
    from jnerf_b200 import ops
    if table not in _LEVELS:
        aabb, log2T, primes = TABLES[table]
        _LEVELS[table] = (ops.HashLevels(aabb, log2_hashmap_size=log2T, primes=primes), ol.HashCfg(aabb, log2_hashmap_size=log2T), primes)
    return _LEVELS[table]


@functools.lru_cache(None)
def _march():
    from test_gpu_network_fwd_reference import _march_rows
    cc, n_dev = _march_rows(21)
    assert int(n_dev.view(torch.int32)[0]) >= N, "the march must fill the 2^18-row batch"
    return cc.cpu().numpy()


@functools.lru_cache(maxsize=8)
def _big(table, rows):
    lv, cfg, primes = _levels(table)
    scales = device_scales(lv)
    x = _march()[:, :3].copy()
    if rows == "faces":
        rng = np.random.default_rng(7)
        x = snap_rows(x[:N - 77], face_values(scales, range(0, L, 3), rng), rng, share=0.2)
    return Geometry(cfg, x, scales, primes), x


def _inputs(table, rows):
    """[(geometry, x)] of a row set"""
    if rows != "small":
        return [_big(table, rows)]
    lv, cfg, primes = _levels(table)
    x = _march()[:max(SMALL), :3].copy()
    return [(Geometry(cfg, x[:n], device_scales(lv), primes), x[:n]) for n in SMALL]


def _grid(cfg, dt, seed):
    rng = np.random.default_rng(seed)
    return (rng.uniform(-1, 1, cfg.n_params) * (1e-4 if dt == np.float16 else 1.0)).astype(dt)    # fp16: the NGP initialisation's range


CASES = [(t, r, d) for t in TABLES for r in ("march", "faces", "small") for d in ("fp32", "fp16")]


@pytest.mark.parametrize("table,rows,dt", CASES, ids=[f"{t}-{r}-{d}" for t, r, d in CASES])
def test_hash_fwd(table, rows, dt):
    from jnerf_b200 import ops
    t0 = time.time()
    lv, cfg, primes = _levels(table)
    dt = np.float16 if dt == "fp16" else np.float32
    bits = np.uint16 if dt == np.float16 else np.uint32
    grid = _grid(cfg, dt, 11)
    rng = np.random.default_rng(12)
    worst, fails = 0.0, []
    for geo, x in _inputs(table, rows):
        n = x.shape[0]
        out = ops.hash_fwd(_cu(x), _cu(grid), lv).cpu().numpy()
        with level_scales(geo.scales, primes):
            ref = ol.hash_fwd(cfg, x, grid, acc32=True)
        bad = np.flatnonzero((out.view(bits) != ref.view(bits)).any(1))
        if bad.size:
            fails.append(f"n={n}: {bad.size} rows differ from the oracle's per-point evaluation, first {bad[:8].tolist()}")
        if n > 1:
            p = rng.permutation(n)
            outp = ops.hash_fwd(_cu(x[p]), _cu(grid), lv).cpu().numpy()
            if not np.array_equal(outp.view(bits)[np.argsort(p)], out.view(bits)):
                fails.append(f"n={n}: a permutation of the rows changed the output")
        if dt == np.float16 and n:
            coords = np.zeros((n, 7), np.float32)
            coords[:, :3], coords[:, 4:] = x, _march()[:n, 4:]
            wrng = np.random.default_rng(13)
            _, enc = ops.network_fwd(_cu(coords), _cu(grid), lv, _cu(mlp_weights(0, wrng)), _cu(mlp_weights(1, wrng)))
            if not np.array_equal(enc.cpu().numpy().view(np.uint16), out.view(np.uint16)):
                fails.append(f"n={n}: the fused forward saved another encoding")
        y, e = hash_fwd_f64(geo, grid, "cuda")
        ok, ratio = check_fwd(out, y, e)
        if not ok.all():
            fails.append(f"n={n}: {int((~ok).sum())} entries outside the fp64 bound, first {np.argwhere(~ok)[:4].tolist()}")
        worst = max(worst, float(ratio.max()) if ratio.size else 0.0)
    print(f"[operator-fp64] hash_fwd {table}/{rows}/{np.dtype(dt).name}: worst error/bound {worst:.3g}; {time.time() - t0:.1f} s")
    assert not fails, fails[:6]


def _run_stats(geo, dy):
    """(zero rows skipped inside a run, paired x-neighbour reductions) of the kernel's partition, over all levels"""
    inside = paired = 0
    for l in range(L):
        rows, run, first = partition(geo, dy, l)
        zero = np.flatnonzero((dy[:, 2 * l] == 0) & (dy[:, 2 * l + 1] == 0))
        p = np.searchsorted(rows, zero) - 1
        ok = (p >= 0) & (p + 1 < rows.size)
        inside += int((run[p[ok]] == run[np.minimum(p[ok] + 1, rows.size - 1)]).sum())
        idx = geo.idx[first, l, :]
        paired += int(sum(((idx[:, c] ^ idx[:, c + 1]) == 1).sum() for c in range(0, 8, 2)))
    return inside, paired


@pytest.mark.parametrize("table,rows,dt", CASES, ids=[f"{t}-{r}-{d}" for t, r, d in CASES])
def test_hash_bwd(table, rows, dt):
    from jnerf_b200 import ops
    t0 = time.time()
    lv, cfg, primes = _levels(table)
    fp16 = dt == "fp16"
    worst, fails, rep = 0.0, [], ""
    for geo, x in _inputs(table, rows):
        n = x.shape[0]
        dy = training_dy(n, np.random.default_rng(n + 3), fp16)
        got = ops.hash_bwd(_cu(x), _cu(dy), lv).cpu().numpy()
        with level_scales(geo.scales, primes):
            g, a, cnt = ol.hash_bwd_f64(cfg, x, dy.astype(np.float32))
        R, mean_run = reductions(geo, dy)
        n_out, n_untouched, w, tight = check_bwd(got, g, a, cnt, R, fp16)
        worst = max(worst, w)
        if n_out or n_untouched:
            fails.append(f"n={n}: {n_out} entries outside the bound, {n_untouched} entries no row reaches are nonzero")
        if rows != "small":
            inside, paired = _run_stats(geo, dy)
            nzg = got[got != 0].astype(np.float64)
            sub = float((np.abs(nzg) < 2.0 ** -14).mean()) if fp16 and nzg.size else 0.0
            rep = (f"; level-0 rows per run {mean_run[0]:.2f} (level 15: {mean_run[-1]:.2f}), {inside} zero rows inside runs, {paired} paired "
                   f"reductions, subnormal share {sub:.3f}, bound < 1 % of A_e on {tight:.3f} of {int((cnt > 0).sum())} touched")
            if not (mean_run[0] > 4 and inside > 0 and (paired > 0 or not fp16)):
                fails.append(f"the inputs do not exercise the runs: {rep}")
    print(f"[operator-fp64] hash_bwd {table}/{rows}/{dt}: worst error/bound {worst:.3g}{rep}; {time.time() - t0:.1f} s")
    assert not fails, fails[:6]


@pytest.mark.parametrize("dt", ["fp32", "fp16"])
def test_sh(dt):
    from jnerf_b200 import ops
    d = np.concatenate([sh_special_directions(np.random.default_rng(17)), _march()[:, 4:]])[:N]
    out = ops.sh_fwd(_cu(d), torch.float16 if dt == "fp16" else torch.float32).cpu().numpy()
    want = sh_f32(d, contract=True)
    if dt == "fp16":
        want = want.astype(np.float16)
        lo, hi = (t.numpy() for t in sh_interval(d))
        o = out.astype(np.float64)
        inside = (o >= lo) & (o <= hi)
    else:
        v, e = (t.numpy() for t in sh_f64(d))
        inside = np.abs(out.astype(np.float64) - v) <= e
    bits = np.uint16 if dt == "fp16" else np.uint32
    diff = np.argwhere(out.view(bits) != want.view(bits))
    print(f"[operator-fp64] sh {dt}: {d.shape[0]} directions, {int((~inside).sum())} outside the interval, {diff.shape[0]} differ from sh_f32")
    assert inside.all() and diff.shape[0] == 0, (np.argwhere(~inside)[:4].tolist(), diff[:4].tolist())


MLP_CASES = [(h, n) for h in range(4) for n in (1, 127, 129, N - 77, N)]


@pytest.mark.parametrize("nhm,n", MLP_CASES, ids=[f"nhm{h}-{n}" for h, n in MLP_CASES])
def test_mlp(nhm, n):
    from jnerf_b200 import ops
    t0 = time.time()
    sm = int(ops.lib.load().ngp_sm_count())
    k_cta, n_cta = mlp_bwd_ctas(n, nhm, sm)
    tiles = (n + 127) // 128
    fwd_tiles = -(-tiles // min(tiles, 4 * sm))
    rep, fails = [], []
    for probe in (False, True):
        rng = np.random.default_rng(nhm * 7 + n)
        W = mlp_probe_weights(nhm) if probe else mlp_weights(nhm, rng)
        X = np.clip(rng.standard_normal((n, 32)), -4, 4).astype(np.float16)
        nv = 16 if nhm == 0 else 3
        dY = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
        dY[:, nv:] = 0
        Wt, Xt, dYt = _cu(W), _cu(X), _cu(dY)
        Y, inter = ops.mlp_fwd(Wt, Xt, nhm)
        dX, temps, dW = ops.mlp_bwd(Wt, Xt, inter, dYt, nhm, nv, need_dx=True, need_temps=True)
        dX2, temps2 = ops.mlp_bwd_dgrad(Wt, inter, dYt.T.contiguous(), nhm, need_dx=True)
        torch.cuda.synchronize()
        assert ops.lib.load().ngp_debug_timeout_flag() == 0
        worst, f = check_mlp(Wt, Xt, inter, Y, dYt, temps, dX, dW, nhm, nv, k_cta, n_cta)
        tag = "probe" if probe else "realistic"
        fails += [f"{tag}: {s}" for s in f]
        b = lambda t: t.view(torch.int16)
        if not (torch.equal(b(temps2), b(temps)) and torch.equal(b(dX2), b(dX))):
            fails.append(f"{tag}: the feature-major dgrad differs from ngp_mlp_bwd")
        if probe:
            if not torch.equal(Y[:, :16], Xt[:, :16]):
                fails.append("probe: Y is not the routed input")
            if not torch.equal(dX[:, :16], torch.where(Xt[:, :16] != 0, dYt, torch.zeros_like(dYt))) or bool((dX[:, 16:] != 0).any()):
                fails.append("probe: dX is not the routed output gradient")
        rep.append(f"{tag} " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    print(f"[operator-fp64] mlp nhm={nhm} n={n}: forward tiles per CTA {fwd_tiles}, backward rows per CTA {k_cta} over {n_cta} CTAs; "
          f"worst error/bound {'; '.join(rep)}; {time.time() - t0:.1f} s")
    if n == N:
        assert fwd_tiles > 1
    assert not fails, fails[:6]
