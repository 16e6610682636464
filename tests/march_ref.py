"""Restatements and bounds shared by the march and occupancy-grid tests (test_march_bound_cpu.py on the CPU,
test_gpu_march_reference.py and test_gpu_grid_update_reference.py on the GPU).

  * closed_form / sequential: the const_dt shortcut of march_count_kernel's stage1 (csrc/sampler.cu) in numpy float32, and the
    sequential float additions it replaces;
  * mean_f32 / mean_f64 / mean_bound: mean_partial_kernel + mean_final_kernel (csrc/grid_update.cu) emulated in float32, the exact
    mean, and the bound of the fixed-order reduction;
  * splat_bound: the per-entry bound of splat_kernel's __expf(x) * sqrt(3)/1024 against float64;
  * n_emit / row_t / step_of_rows / chunk_crosses_binade: the march workspace's per-ray emitting-chunk counts, the ray parameter t
    recovered from an emitted row, the const_dt step that row belongs to, and which 32-step chunks cross a power of two."""
import numpy as np

G3 = 128 ** 3
U = 2.0 ** -24                                                   # unit roundoff of float32
MIN_CONE = np.float32(np.float32(1.73205080757) / np.float32(1024))
H_CONST = np.float32(MIN_CONE * np.float32(0.5))                 # calc_dt with const_dt: MIN_CONE_STEPSIZE() * 0.5
THICK = float(np.float32(np.float32(1.73205080757) / np.float32(1024.0)))   # the fp32 constant splat_kernel multiplies by


def gamma(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------- const_dt closed form
def _fma32(a, b, c):
    """fl32(a * b + c) for the operands the closed form uses: a * b and the sum are exact in float64 (a < 64, b a multiple of ulp(c)
    or smaller than c by < 2^29), so one rounding to float32 is the fused multiply-add."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


MUTANTS = ("no_tie", "window_116", "window_141", "no_e1")


def closed_form(tc, h=H_CONST, mutant=None):
    """stage1's shortcut for chunk starts tc (float32, > 0): (taken mask, the 32 lane values t_k, t of the next chunk)."""
    assert mutant in (None, *MUTANTS), mutant
    tc = np.ascontiguousarray(tc, np.float32)
    h = np.float32(h)
    q = (tc + h) - tc                                            # exact (Sterbenz)
    t_end = _fma32(32.0, q, tc)
    e0 = (tc.view(np.uint32) >> 23).astype(np.int64)
    e1 = (t_end.view(np.uint32) >> 23).astype(np.int64)
    lo = 116 if mutant == "window_116" else 117
    hi = 141 if mutant == "window_141" else 140
    in_window = (e0 >= lo) & (e0 <= hi)
    scale = (np.where(in_window, 277 - e0, 127).astype(np.uint32) << 23).view(np.float32)
    r = h * scale                                                # h / ulp(tc), exact
    tie = (r - np.floor(r)) == np.float32(0.5)
    if mutant == "no_tie":
        tie = np.zeros_like(tie)
    same = (e0 == e1) if mutant != "no_e1" else np.ones_like(in_window)
    taken = same & in_window & ~tie
    lanes = _fma32(np.arange(32, dtype=np.float64)[None, :], q[:, None], tc[:, None])
    return taken, lanes, t_end


def sequential(tc, h=H_CONST, n=33):
    """t_0 .. t_{n-1} of t_{k+1} = fl32(t_k + h): what the reference's loop (and the kernel's fallback) computes."""
    t = np.ascontiguousarray(tc, np.float32).copy()
    h = np.float32(h)
    out = np.empty((t.size, n), np.float32)
    for k in range(n):
        out[:, k] = t
        t = t + h
    return out


def closed_form_mismatches(tc, h=H_CONST, mutant=None):
    """Chunk starts where the shortcut is taken and differs from the sequential additions in any lane or in the next chunk's start."""
    taken, lanes, t_end = closed_form(tc, h, mutant)
    seq = sequential(tc, h)
    bad = taken & ((lanes.view(np.uint32) != seq[:, :32].view(np.uint32)).any(1) | (t_end.view(np.uint32) != seq[:, 32].view(np.uint32)))
    return bad, taken


# ---------------------------------------------------------------------------------------------------- grid mean
def mean_f64(grid):
    """The exact mean of cascade 0: sum of fl32(max(g, 0) / G3) in float64 (orc_grid_mean before its final rounding)."""
    a = (np.maximum(grid[:G3].astype(np.float32), np.float32(0)) / np.float32(G3)).astype(np.float64)
    return float(a.sum()), a


def mean_bound(grid):
    """|fp32 reduction - mean_f64| for mean_partial_kernel / mean_final_kernel.  Every addend is >= 0, so a chain of d roundings bounds
    the error by gamma(d) * sum: 31 serial additions per thread (32 addends, the first onto 0 is exact), an 8-level tree over 256
    threads, an 8-level tree over 256 blocks -- d = 47.  Addends below 2^-126 may each carry one more subnormal rounding, 2^-150."""
    s, a = mean_f64(grid)
    n_sub = int(np.count_nonzero((a > 0) & (a < 2.0 ** -126)))
    return gamma(31 + 8 + 8) * s + n_sub * 2.0 ** -150


def mean_f32(grid, serial=32):
    """mean_partial_kernel + mean_final_kernel in float32, operation for operation: 256 blocks of 8192 cells, thread t of a block adds
    cells t, t + 256, ... in order, then two 256-wide trees (s[t] += s[t + off], off = 128 .. 1).  `serial` other than 32 restates a
    different split of a block (serial adds per thread, 8192 / serial threads) -- a reordering the bound above does not cover."""
    a = np.maximum(grid[:G3].astype(np.float32), np.float32(0)) / np.float32(G3)
    threads = 8192 // serial
    blk = a.reshape(256, serial, threads)
    acc = np.zeros((256, threads), np.float32)
    for j in range(serial):
        acc = acc + blk[:, j, :]
    s = acc
    while s.shape[1] > 1:
        half = s.shape[1] // 2
        s = s[:, :half] + s[:, half:2 * half]
    p = s[:, 0].copy()
    while p.size > 1:
        half = p.size // 2
        p = p[:half] + p[half:]
    return np.float32(p[0])


# ---------------------------------------------------------------------------------------------------- splat
def expf_ulps(x):
    """__expf's maximum error in ulps (CUDA C Programming Guide, intrinsic functions): 2 + floor(|1.173 x|)."""
    return 2.0 + np.floor(1.173 * np.abs(np.asarray(x, np.float64)))


def ulp32(y):
    """ulp of a float32 of magnitude y (subnormal spacing 2^-149 below 2^-126)."""
    y = np.abs(np.asarray(y, np.float64))
    e = np.floor(np.log2(np.maximum(y, 2.0 ** -126)))
    return np.exp2(np.maximum(e - 23, -149))


def splat_ref(x):
    """float64 exp(x) * THICK and its bound for fl32(THICK * __expf(x)): __expf's ulp error, then the product's one rounding
    (relative 2^-24, or half a subnormal step)."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore"):
        e = np.exp(x)
        ref = e * THICK
        err_exp = expf_ulps(x) * ulp32(e)
        bound = THICK * err_exp + U * THICK * (e + err_exp) + 2.0 ** -150
    return ref, bound


# ---------------------------------------------------------------------------------------------------- march workspace / rows
def n_emit(workspace, n_rays):
    """Emitting-chunk count per ray from ngp_march's workspace: counts[R] | n_emit[R] | 256-aligned chunk records (uint32 each)."""
    w = np.asarray(workspace)
    assert w.dtype == np.uint8 and w.size >= 8 * n_rays
    return w[:8 * n_rays].view(np.uint32)[n_rays:2 * n_rays].copy()


def row_t(rows, rays_o, rays_d, aabb):
    """The ray parameter t of emitted rows (q = (fma(t, d, o) - lo) / (hi - lo)): p recovered in float64 and t read off the component
    with the largest |d|.  Accurate to a few ulp of p over |d| >= 1/sqrt(3): enough to place t in a binade away from its edges."""
    lo, hi = float(aabb[0]), float(aabb[1])
    p = rows[:, :3].astype(np.float64) * (hi - lo) + lo
    o = np.asarray(rays_o, np.float64)
    d = np.asarray(rays_d, np.float64)
    k = np.argmax(np.abs(d), axis=1)
    r = np.arange(len(k))
    return (p[r, k] - o[r, k]) / d[r, k]


def step_of_rows(t_rows, ray_of_row, seq):
    """Index k of the step t_k = seq[ray, k] nearest to each row's recovered t (rows of one ray in increasing t), and the largest
    |t_row - t_k| -- far below the step when the recovery is right."""
    k = np.empty(t_rows.size, np.int64)
    bounds = np.r_[0, np.flatnonzero(np.diff(ray_of_row)) + 1, t_rows.size]
    for b, e in zip(bounds[:-1], bounds[1:]):
        s = seq[ray_of_row[b]].astype(np.float64)
        j = np.clip(np.searchsorted(s, t_rows[b:e]), 1, s.size - 1)
        k[b:e] = np.where(np.abs(s[j - 1] - t_rows[b:e]) <= np.abs(s[j] - t_rows[b:e]), j - 1, j)
    return k, float(np.abs(seq[ray_of_row, k].astype(np.float64) - t_rows).max()) if t_rows.size else 0.0


def chunk_crosses_binade(seq):
    """(R, C): whether chunk c of each ray (steps 32c .. 32c + 31 of seq) has its first and last t in different binades -- a chunk the
    closed form must leave to the sequential additions."""
    R, n = seq.shape
    C = n // 32
    e = seq[:, :32 * C].view(np.uint32) >> 23
    return e[:, 0::32] != e[:, 31::32]
