"""Float64 references and per-entry error bounds of the per-operator NGP kernels: the hash-grid forward and backward and the SH encoder
(csrc/hash_encode.cu) and the fully-fused MLP (csrc/mlp_tc.cu), with host models of their arithmetic for the CPU rehearsal.

Hash-grid geometry.  hash_cell forms p = fmaf(x, scale, 0.5) per dimension, the cell g = floor(p) and the fraction f = p - g (exact), and
hash_cell_weights the corner weights w_c = ((1 * wx) * wy) * wz, wx = {1 - f, f}, each step an fp32 rounding.  Geometry reproduces these
bit for bit (ngp_fwd_ref.fma32 is a correctly rounded fp32 fma); corner indices come from the oracle (orc_hash_indices), with the level
scales installed from the same fp32 array (level_scales) so that host and kernel agree on every cell.

Forward bound.  Each feature is an fmaf chain over the 8 corners, so its fp32 value lies within gamma_8 sum_c |w_c v_c| (+ 8 halves of the
smallest fp32 subnormal) of the exact sum_c w_c v_c (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 3.1); the
fp16 table's output is one rounding of that fp32 value.

Backward partition.  hash_bwd_kernel gives thread (block, sub) the RUN consecutive rows [RUN k, RUN k + RUN) of a chunk k at every level.
It skips rows whose two features of the level have zero gradient, starts a new run when a row lands in another cell than the previous
non-skipped row of the chunk, sums dy * w_c per corner in fp32 (one fmaf per row) and flushes each run's 8 corner sums with one reduction
each: red.add.v2.f32, or fp16 -- two x-neighbour entries that share an aligned word in one red.add.v2.f16x2 (red_add_corners).
partition() reproduces that split; R_e, the number of reductions that reach entry e, is the number of (run, corner) pairs whose corner
index is e.  It is a model of the kernel's partition, not an upper bound of it: if the kernel's RUN, its chunking or its run-start rule
changes, partition() and the bounds that use it must change with it (RUN is read from the source).  cnt_e, the number of non-zero
contributions, also bounds R_e but makes the fp16 bound vacuous at the coarse levels, where one entry collects thousands of rows.

Backward bound, per feature of entry e with exact sum g_e and sum of |terms| A_e (oracle orc_hash_bwd_f64):
- a run of at most RUN terms summed by fmaf is off by at most gamma_RUN (sum of its |terms|): gamma_RUN A_e over all runs;
- fp32: the R_e run sums are added by fp32 atomics in some order, recursive summation: gamma_{R_e} (1 + gamma_RUN) A_e;
- fp16: each run sum is rounded to fp16 once, u16 |s| + 2^-25 (2^-25 is half the smallest subnormal: no flush to zero), and each atomic
  add rounds its partial sum: gamma16_{R_e} of the sum of the rounded run values plus 2^-25 per add.
An entry that no row reaches must hold exactly 0.

MLP.  Each layer is checked from the kernel's own stored operands, as nerf_mlp_ref does: every stored fp16 value is a correct rounding of a
value within the fwd_layer / dgrad_layer accumulation bound (tensor-core alignment floor included) of the exact product, ReLU clamped
first; a backward block is zero where the forward's stored activation is not positive.  Weight gradients accumulate a CTA's rows in
fp32 tensor-core registers across its tiles, then add the CTAs' fragments with fp32 reductions in any order: (K + C + 2) 2^-23 (sum |term|
+ F) bounds that for K rows per CTA and C CTAs."""
import os
import re

import numpy as np
import torch

import oracle_lib as ol
from ngp_fwd_ref import fma32
from nerf_mlp_ref import U, _floor, check_rounding, dgrad_layer, fwd_layer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32, U16 = 2.0 ** -24, 2.0 ** -11
ETA32, ETA16 = 2.0 ** -150, 2.0 ** -25          # half the smallest fp32 / fp16 subnormal
L = 16
DEFAULT_PRIMES = (1, 19349663, 83492791)
IN, WIDTH, OUTP = 32, 64, 16


def _hash_run():
    """RUN of hash_encode.cu, and a check that a block still covers (HASH_THREADS / N_LEVELS) * RUN consecutive rows"""
    src = open(os.path.join(ROOT, "jnerf_b200", "csrc", "hash_encode.cu")).read()
    run = int(re.search(r"constexpr int RUN = (\d+);", src).group(1))
    assert "RUN_PTS_PER_BLOCK = (HASH_THREADS / N_LEVELS) * RUN;" in src and "base = blockIdx.x * RUN_PTS_PER_BLOCK + sub * RUN;" in src, \
        "the backward's row partition changed: update partition()"
    return run


RUN = _hash_run()


def gamma(k, u):
    """k u / (1 - k u), inf where k u >= 1 (no bound)"""
    k = np.asarray(k, np.float64)
    ku = k * u
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ku < 1, ku / (1 - ku), np.inf)


def host_scales(cfg):
    """fp32 level scales exp2f(l log2_pls) * base - 1 on the host (the GPU tests use the device's, level_scales(device_scales(lv)))"""
    l = np.arange(L, dtype=np.float32)
    return (np.exp2(l * np.float32(cfg.log2_pls)).astype(np.float32) * np.float32(cfg.base) - np.float32(1)).astype(np.float32)


def device_scales(lv):
    return np.ascontiguousarray(lv.table.cpu().numpy().view(np.float32).reshape(L, 8)[:, 0])


class level_scales:
    """Install fp32 level scales (and optionally hash primes) into the oracle for the duration of a block."""

    def __init__(self, scales, primes=DEFAULT_PRIMES):
        self.scales, self.primes = np.ascontiguousarray(scales, np.float32), tuple(primes)

    def __enter__(self):
        ol.oracle().orc_set_level_scales(ol._ptr(self.scales))
        ol.oracle().orc_set_hash_primes(*self.primes)

    def __exit__(self, *a):
        ol.oracle().orc_set_level_scales(None)
        ol.oracle().orc_set_hash_primes(*DEFAULT_PRIMES)


# ---------------------------------------------------------------------------------------------------------------- hash grid
class Geometry:
    """Per level of fp32 points x (n, 3): cells (L, n, 3) int32, corner weights w (L, n, 8) float32 exactly as the kernels form them, and
    the oracle's global corner entry indices idx (n, L, 8)."""

    def __init__(self, cfg, x, scales, primes=DEFAULT_PRIMES):
        x = np.ascontiguousarray(x, np.float32)
        n = x.shape[0]
        self.n, self.cfg, self.scales, self.primes = n, cfg, scales, primes
        self.cells = np.empty((L, n, 3), np.int32)
        self.w = np.empty((L, n, 8), np.float32)
        one = np.float32(1)
        for l in range(L):
            p = fma32(x, scales[l], np.float32(0.5))
            g = np.floor(p)
            f = (p - g).astype(np.float32)
            self.cells[l] = g.astype(np.int32)
            wd = [(one - f[:, d], f[:, d]) for d in range(3)]
            for c in range(8):
                self.w[l, :, c] = ((one * wd[0][c & 1]) * wd[1][(c >> 1) & 1]) * wd[2][(c >> 2) & 1]
        with level_scales(scales, primes):
            self.idx = ol.hash_indices(cfg, x)


def hash_fwd_f64(geo, grid, device="cpu"):
    """(y, e) (n, 32) float64 tensors on `device`: the exact sum_c w_c v_c per feature and the bound of the kernel's fp32 fmaf chain"""
    g2 = torch.as_tensor(np.asarray(grid).reshape(-1, 2).astype(np.float64), device=device)
    idx = torch.as_tensor(geo.idx.astype(np.int64), device=device)
    w = torch.as_tensor(geo.w, device=device).to(torch.float64).permute(1, 0, 2)
    t = w[..., None] * g2[idx]                                # (n, L, 8, 2): every product exact in float64
    return t.sum(2).reshape(geo.n, 2 * L), float(gamma(8, U32)) * t.abs().sum(2).reshape(geo.n, 2 * L) + 8 * ETA32


def check_fwd(out, y, e):
    """(ok, ratio) numpy of the kernel's fp32 or fp16 output (numpy) against the exact sum y and the fp32 bound e (tensors on one device;
    fp16: a rounding of the fp32 value)"""
    got = torch.as_tensor(np.asarray(out), device=y.device)
    if got.dtype == torch.float16:
        ok, ratio = check_rounding(got, y, e)
    else:
        err = (got.to(torch.float64) - y).abs()
        ok, ratio = err <= e, torch.where(err > 0, err / e, torch.zeros_like(err))
    return ok.cpu().numpy(), ratio.cpu().numpy()


def partition(geo, dy, level, merge_z=False):
    """The backward's runs at one level: (rows, run) of the rows it does not skip, run ids in order, and the first row of every run.
    merge_z: the run-start rule of a kernel that ignores gz (a mutant of the CPU rehearsal)."""
    nz = (dy[:, 2 * level] != 0) | (dy[:, 2 * level + 1] != 0)
    rows = np.flatnonzero(nz)
    c = geo.cells[level, rows][:, :2 if merge_z else 3]
    chunk = rows // RUN
    new = np.ones(rows.size, bool)
    new[1:] = (chunk[1:] != chunk[:-1]) | (c[1:] != c[:-1]).any(1)
    return rows, np.cumsum(new) - 1, rows[new]


def reductions(geo, dy):
    """R_e (n_entries,) int64: the number of reductions of the kernel's partition that reach each entry, and per level the mean number of
    rows per run"""
    ents, mean_run = [], []
    for l in range(L):
        rows, run, first = partition(geo, dy, l)
        ents.append(geo.idx[first, l, :].ravel())
        mean_run.append(rows.size / max(first.size, 1))
    return np.bincount(np.concatenate(ents), minlength=geo.cfg.n_entries), np.array(mean_run)


def hash_bwd_bound(a, R, fp16, run=RUN):
    """The per-feature bound of the module docstring from A_e (n_params,) and R_e (n_params,); run: the longest fmaf run"""
    g_run = gamma(run, U32)
    s = (1 + g_run) * a                                   # >= the sum of |fp32 run sums|
    if not fp16:
        return g_run * a + gamma(R, U32) * s + (R + run) * ETA32
    h = (1 + U16) * s + R * ETA16                          # >= the sum of |fp16 run values|
    return g_run * a + U16 * s + R * ETA16 + gamma(R, U16) * h + R * ETA16


def check_bwd(got, g, a, cnt, R, fp16):
    """(n_outside, n_written_untouched, worst ratio, share of touched entries whose bound is below 1 % of A_e)"""
    got = np.asarray(got)
    t = np.flatnonzero(cnt)
    bound = hash_bwd_bound(a[t], R[t // 2], fp16)
    err = np.abs(got[t].astype(np.float64) - g[t])
    ratio = err / np.maximum(bound, 1e-300)
    n_untouched = int(np.count_nonzero(got)) - int(np.count_nonzero(got[t]))
    return (int((err > bound).sum()), n_untouched, float(ratio.max()) if t.size else 0.0,
            float((bound < 0.01 * a[t]).mean()) if t.size else 0.0)


def model_hash_bwd(geo, dy, fp16, rng, mutant=None):
    """A numpy model of hash_bwd_kernel: the partition, per-run fp32 fmaf sums, (fp16: one rounding per run, red_add_corners' pairing)
    and the reductions applied in a random order, one correctly rounded add at a time.  mutant: None, "swap-halves" (the two halves of a
    paired x-neighbour reduction exchanged), "drop-last-run" (the last run of every chunk never flushed), "stale-gz" (a run continues when
    only gz changes, keeping its corner indices), "ftz" (fp16 subnormal run sums flushed to zero)."""
    d32 = np.asarray(dy, np.float32)
    ents, vals = [], []
    for l in range(L):
        rows, run, first = partition(geo, d32, l, merge_z=mutant == "stale-gz")
        nrun = first.size
        acc = np.zeros((nrun, 8, 2), np.float32)
        pos = rows % RUN
        for k in range(RUN):
            sel = pos == k
            r, j = rows[sel], run[sel]
            acc[j] = fma32(d32[r, None, 2 * l:2 * l + 2], geo.w[l, r, :, None], acc[j])
        idx = geo.idx[first, l, :].astype(np.int64)
        if mutant == "drop-last-run":
            last = np.ones(nrun, bool)
            last[:-1] = first[1:] // RUN != first[:-1] // RUN
            acc, idx = acc[~last], idx[~last]
        if fp16:
            v = acc.astype(np.float16)
            if mutant == "ftz":
                v = np.where(np.abs(v) < np.float16(2.0 ** -14), np.float16(0), v)
            if mutant == "swap-halves":
                for c in range(0, 8, 2):
                    pair = (idx[:, c] ^ idx[:, c + 1]) == 1
                    v[pair, c], v[pair, c + 1] = v[pair, c + 1].copy(), v[pair, c].copy()
        else:
            v = acc
        ents.append(np.repeat(idx.ravel(), 2) * 2 + np.tile([0, 1], idx.size))
        vals.append(v.reshape(-1))
    ent, val = np.concatenate(ents), np.concatenate(vals)
    order = np.lexsort((rng.random(ent.size), ent))
    ent, val = ent[order], val[order]
    start = np.flatnonzero(np.r_[True, ent[1:] != ent[:-1]])
    rank = np.arange(ent.size) - np.repeat(start, np.diff(np.r_[start, ent.size]))
    by_rank = np.argsort(rank, kind="stable")                 # the k-th reduction of every entry, k = 0, 1, ..., as one slice each
    ent, val, rank = ent[by_rank], val[by_rank], rank[by_rank]
    cut = np.searchsorted(rank, np.arange(int(rank.max()) + 2 if rank.size else 1))
    out = np.zeros(geo.cfg.n_params, np.float16 if fp16 else np.float32)
    for k0, k1 in zip(cut[:-1], cut[1:]):
        e, v = ent[k0:k1], val[k0:k1]
        if fp16:
            out[e] = (out[e].astype(np.float64) + v.astype(np.float64)).astype(np.float16)   # exact in float64, one rounding
        else:
            out[e] = out[e] + v
    return out


def face_values(scales, levels, rng, per_level=64):
    """fp32 coordinates in [0, 1] where fmaf(x, scale, 0.5) is an integer (a cell face) at each of `levels`"""
    out = []
    for l in levels:
        s = np.float32(scales[l])
        k = np.arange(1, int(s) + 1, dtype=np.float64)
        c = ((k - 0.5) / np.float64(s)).astype(np.float32)
        cand = np.concatenate([c, np.nextafter(c, np.float32(0)), np.nextafter(c, np.float32(1))])
        cand = cand[(cand >= 0) & (cand <= 1)]
        p = fma32(cand, s, np.float32(0.5))
        hit = cand[p == np.floor(p)]
        assert hit.size, f"no face found at level {l}"
        out.append(rng.choice(hit, min(per_level, hit.size), replace=False))
    return np.concatenate(out)


def snap_rows(x, faces, rng, share=0.3):
    """x with a share of its 8-row blocks given one coordinate on a face, at 0 or at 1, the same for the whole block, so runs stay"""
    x = x.copy()
    n = x.shape[0]
    nb = (n + 7) // 8
    blk = np.arange(n) // 8
    vals = np.concatenate([faces, np.float32([0, 1] * max(1, faces.size // 8))])
    pick, v, d = rng.random(nb) < share, rng.choice(vals, nb), rng.integers(0, 3, nb)
    rows = np.flatnonzero(pick[blk])
    x[rows, d[blk[rows]]] = v[blk[rows]]
    return x


def training_dy(n, rng, fp16):
    """dL/denc (n, 32) like a training step's: magnitudes from 1e-8 to 1e-3 (most fp16 values subnormal), runs of 3 zero rows every 7
    rows and 5 % single zero rows, and 5 % of the (row, level) pairs with one feature zero"""
    d = rng.standard_normal((n, 2 * L)) * 10.0 ** rng.uniform(-8, -3, (n, 1))
    d[((np.arange(n) // 3) % 7) == 0] = 0
    d[rng.random(n) < 0.05] = 0
    one = rng.random((n, L)) < 0.05
    f = rng.integers(0, 2, (n, L))
    r, l = np.nonzero(one)
    d[r, 2 * l + f[r, l]] = 0
    return d.astype(np.float16 if fp16 else np.float32)


# ---------------------------------------------------------------------------------------------------------------- SH
def sh_special_directions(rng, m=4096):
    """Encoded directions (components in [0, 1], x = 2 d - 1) where sh4 is hardest to evaluate: the 6 axes, the 8 cube diagonals, every
    component combination of 0, 0.5 and 1, and m directions each for the cancelling differences 1 - 5 z^2 and 5 z^2 - 3 (z near +-1/sqrt5,
    +-sqrt(3/5)), x^2 - y^2 (|x| = |y|), -3 x^2 + y^2 (|y| = sqrt3 |x|) and -x^2 + 3 y^2 (|x| = sqrt3 |y|), the cancelling component
    nudged by -3 .. 3 fp32 ulps."""
    d = [np.eye(3), -np.eye(3), np.array(np.meshgrid([-1, 1], [-1, 1], [-1, 1], indexing="ij")).reshape(3, -1).T / np.sqrt(3)]
    enc = [((np.concatenate(d) + 1) / 2).astype(np.float32),
           np.array(np.meshgrid([0, 0.5, 1], [0, 0.5, 1], [0, 0.5, 1], indexing="ij"), np.float32).reshape(3, -1).T]
    nudge = lambda v: _ulps(v, rng.integers(-3, 4, v.shape))
    u = lambda k: rng.uniform(-1, 1, k)
    sgn = lambda k: rng.choice([-1.0, 1.0], k)
    for root in (1 / np.sqrt(5), np.sqrt(0.6)):
        x = np.stack([u(m), u(m), sgn(m) * root], 1)
        e = ((x + 1) / 2).astype(np.float32)
        e[:, 2] = nudge(e[:, 2])
        enc.append(e)
    for a, b, ratio in ((0, 1, 1.0), (1, 0, np.sqrt(3)), (0, 1, np.sqrt(3))):   # |x_b| = ratio |x_a|
        x = np.stack([u(m), u(m), u(m)], 1)
        x[:, a] /= ratio
        x[:, b] = sgn(m) * ratio * x[:, a]
        e = ((x + 1) / 2).astype(np.float32)
        e[:, b] = nudge(e[:, b])
        enc.append(e)
    return np.clip(np.concatenate(enc), 0, 1).astype(np.float32)


def _ulps(v, k):
    """positive fp32 values v moved by k ulps (k may be negative); zeros stay"""
    v = np.ascontiguousarray(v, np.float32)
    return np.where(v > 0, (v.view(np.int32) + k.astype(np.int32)).view(np.float32), v)


# ---------------------------------------------------------------------------------------------------------------- MLP
def mlp_weights(nhm, rng):
    shapes = [(WIDTH, IN)] + [(WIDTH, WIDTH)] * nhm + [(OUTP, WIDTH)]
    lim = lambda s: np.sqrt(6.0 / (s[0] + s[1]))
    return np.concatenate([rng.uniform(-lim(s), lim(s), s).astype(np.float16).ravel() for s in shapes])


def mlp_probe_weights(nhm):
    """W0 = [I32; -I32], every hidden matmul the identity, Wout row j = e_j - e_{32+j}: inter_0 = [relu(X) | relu(-X)], Y[:, j] = X[:, j]
    and dX[:, j] = dY[:, j] where X[:, j] != 0 (j < 16), every product and sum exact in fp16."""
    w0 = np.zeros((WIDTH, IN), np.float16)
    w0[np.arange(IN), np.arange(IN)] = 1
    w0[IN + np.arange(IN), np.arange(IN)] = -1
    wo = np.zeros((OUTP, WIDTH), np.float16)
    wo[np.arange(OUTP), np.arange(OUTP)] = 1
    wo[np.arange(OUTP), IN + np.arange(OUTP)] = -1
    return np.concatenate([w0.ravel()] + [np.eye(WIDTH, dtype=np.float16).ravel()] * nhm + [wo.ravel()])


def split_mlp(W, nhm):
    """(W0 (64, 32), [Wh_k (64, 64)], Wout (16, 64)) float64 of a flat weight tensor"""
    W = W.to(torch.float64)
    o = WIDTH * IN
    wh = [W[o + k * WIDTH * WIDTH:o + (k + 1) * WIDTH * WIDTH].view(WIDTH, WIDTH) for k in range(nhm)]
    return W[:o].view(WIDTH, IN), wh, W[o + nhm * WIDTH * WIDTH:].view(OUTP, WIDTH)


def mlp_bwd_ctas(n, nhm, sm):
    """(rows per CTA, CTAs) of ngp_mlp_bwd's launch: two CTAs per SM when BwdLayout::total() fits 110 KB"""
    gb = 128 * 16
    total = (4 + 8 * (nhm + 1) + 2 + 8 * (nhm + 1) + 8) * gb + 2 * (WIDTH * IN + nhm * WIDTH * WIDTH + OUTP * WIDTH)
    tiles = (n + 127) // 128
    grid = min(tiles, sm * (2 if total <= 110 * 1024 else 1))
    return 128 * -(-tiles // max(grid, 1)), grid


def check_mlp(W, X, inter, Y, dY, temps, dX, dW, nhm, n_out_valid, k_cta, n_cta):
    """Every stored tensor of one ngp_mlp_fwd + ngp_mlp_bwd against its layer's float64 value from the kernel's own operands (module
    docstring).  Tensors on any one device.  Returns ({tensor: worst ratio}, [failures])."""
    f64 = lambda t: t.to(torch.float64)
    n = X.shape[0]
    W0, Wh, Wout = split_mlp(W, nhm)
    h = f64(inter).view(nhm + 1, n, WIDTH)
    T = f64(temps).view(nhm + 1, n, WIDTH)
    worst, fails = {}, []

    def rec(name, ok, ratio, extra=None):
        bad = (~ok).nonzero()
        worst[name] = float(ratio.max()) if ratio.numel() else 0.0
        if bad.shape[0]:
            fails.append(f"{name}: {bad.shape[0]} entries outside the bound, first {bad[:4].tolist()}")
        if extra:
            fails.append(f"{name}: {extra}")

    zero = lambda k: torch.zeros(k, dtype=torch.float64, device=W.device)
    ins = [f64(X)] + [h[k] for k in range(nhm)]
    mats = [W0] + Wh
    for k in range(nhm + 1):
        y, e = fwd_layer(ins[k], mats[k], zero(WIDTH))
        rec(f"inter{k}", *check_rounding(h[k], y, e, relu=True))
    y, e = fwd_layer(h[nhm], Wout, zero(OUTP))
    rec("Y", *check_rounding(f64(Y), y, e))

    ups = [f64(dY)] + [T[j] for j in range(nhm)]
    mats_b = [Wout] + [Wh[nhm - j] for j in range(1, nhm + 1)]
    for j in range(nhm + 1):
        y, e = dgrad_layer(ups[j], mats_b[j])
        live = h[nhm - j] > 0
        ok, ratio = check_rounding(T[j], y, e)
        dead = int((T[j][~live] != 0).sum())
        rec(f"temps{j}", ok | ~live, torch.where(live, ratio, torch.zeros_like(ratio)),
            f"{dead} entries nonzero where the activation is not positive" if dead else None)
    y, e = dgrad_layer(T[nhm], W0)
    rec("dX", *check_rounding(f64(dX), y, e))

    dW = f64(dW)
    pairs = [(T[nhm], f64(X), 0)] + [(T[nhm - 1 - k], h[k], WIDTH * IN + k * WIDTH * WIDTH) for k in range(nhm)]
    o = WIDTH * IN + nhm * WIDTH * WIDTH
    pairs.append((f64(dY)[:, :n_out_valid], h[nhm], o))
    ratios = []
    for g, x, off in pairs:
        want, a = g.T @ x, g.abs().T @ x.abs()
        F = _floor(g.abs().amax(0), x.abs().amax(0)) if n else torch.zeros_like(a)
        e = (k_cta + n_cta + 2) * U * (a + F)
        got = dW[off:off + want.numel()].view_as(want)
        err = (got - want).abs()
        ratios.append(float((err / e.clamp_min(1e-300)).max()) if n else 0.0)
        nb = int((err > e).sum())
        if nb:
            fails.append(f"dW at {off}: {nb} entries outside the bound")
    worst["dW"] = max(ratios)
    pad = dW[o + n_out_valid * WIDTH:]
    if bool((pad != 0).any()):
        fails.append(f"dW: {int((pad != 0).sum())} entries of padded output rows (>= {n_out_valid}) are nonzero")
    return worst, fails


def model_mlp(W, X, dY, nhm, n_out_valid, mutant=None):
    """A numpy model of the MLP with fp32 accumulation (float32 matmuls of fp16 operands) and an fp16 rounding wherever the kernel
    stores.  mutant: None, "skip-mask" (the ReLU mask of the first backward hidden block skipped), "drop-tail-tile" (the rows of a partial
    last 128-row tile left out of the weight gradients).  Returns (inter, Y, temps, dX, dW) as numpy arrays."""
    f = lambda a: np.asarray(a, np.float16).astype(np.float32)
    W = np.asarray(W, np.float16)
    n = X.shape[0]
    o = WIDTH * IN
    W0 = f(W[:o]).reshape(WIDTH, IN)
    Wh = [f(W[o + k * WIDTH * WIDTH:o + (k + 1) * WIDTH * WIDTH]).reshape(WIDTH, WIDTH) for k in range(nhm)]
    Wout = f(W[o + nhm * WIDTH * WIDTH:]).reshape(OUTP, WIDTH)
    h = [np.maximum(f(X) @ W0.T, 0).astype(np.float16)]
    for k in range(nhm):
        h.append(np.maximum(f(h[-1]) @ Wh[k].T, 0).astype(np.float16))
    Y = (f(h[-1]) @ Wout.T).astype(np.float16)
    T = [((f(dY) @ Wout).astype(np.float16) * (h[nhm] > 0)).astype(np.float16)]
    for j in range(1, nhm + 1):
        t = (f(T[-1]) @ Wh[nhm - j]).astype(np.float16)
        T.append(t if (mutant == "skip-mask" and j == 1) else (t * (h[nhm - j] > 0)).astype(np.float16))
    dX = (f(T[nhm]) @ W0).astype(np.float16)
    keep = n if mutant != "drop-tail-tile" else n // 128 * 128
    dW = np.zeros(W.size, np.float32)
    dW[:o] = (f(T[nhm][:keep]).T @ f(X[:keep])).ravel()
    for k in range(nhm):
        dW[o + k * WIDTH * WIDTH:o + (k + 1) * WIDTH * WIDTH] = (f(T[nhm - 1 - k][:keep]).T @ f(h[k][:keep])).ravel()
    oo = o + nhm * WIDTH * WIDTH
    dW[oo:oo + n_out_valid * WIDTH] = (f(dY[:keep, :n_out_valid]).T @ f(h[nhm][:keep])).ravel()
    return np.concatenate(h), Y, np.concatenate(T), dX, dW
