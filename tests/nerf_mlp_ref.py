"""A float64 reference of the vanilla NeRF network kernels (csrc/nerf_mlp.cu, nerf_mlp.cuh), one layer at a time.

The kernels keep two per-tile slab buffers: `saved`, every layer's input as the forward stored it, and, in the backward's scratch, `dys`,
every layer's pre-activation gradient.  Both are blocks of [groups][128 rows][8 halfs] per 128-row tile.  decode() turns them into
row-major (rows, 8 * groups) matrices whose columns are:

    saved (S_GROUPS = 316)       dys (D_GROUPS = 320)
    enc_pos    0 ..   63         dY_l       256 l .. 256 l + 255, l < 8
    h_l        64 + 256 l        layer 8    2048: [dalpha, 0 x 15, df (256), 0 x 48]
    f          2112 .. 2367      dY9        2368 .. 2495
    enc_dir    2368 .. 2399      dY10       2496: [drgb, 0 x 61]
    v          2400 .. 2527

Each layer is then recomputed exactly from the kernel's own fp16 operands and fp16 weights, so one layer's check does not depend on the
rounding of the layers before it.  The kernel's fp16 result must be a correct rounding of some value within the accumulation bound e of
the exact one: a value in [rn16(y - e), rn16(y + e)] (both ends clamped at 0 first after a ReLU).  rn16 rounds the float64 value to
fp16 once; going through fp32 would round twice and move ties.

The accumulation bound of a K-term dot product plus a bias is e = (K + 2) 2^-23 (sum_k |x_k w_k| + |b| + F), F = 2^-12 max(max_k |x_k|,
max_k |w_k|).  The first term allows every step of an fp32 accumulator to truncate rather than round.  F is the H100 tensor core's
floor: it aligns the products of a k-block at an exponent that does not go below that of a product with a zero (or subnormal) fp16
operand, as if that operand were 2^-14, so a sum far below 2^-14 times its other operands keeps fewer than 24 bits.  Measured on an
H100: a weight-gradient entry of two terms, 8.3e-9 + 3.5e-8, from fp16-subnormal output gradients on rows whose neighbours in the
k-block carry zero gradient and activations near 2, came back truncated to a multiple of 2^-40 (16 significant bits), 1.6 times the
bound without F.  F allows 2^-14 of the largest operand, twice (the mantissa, and a second truncation of the accumulator), on every
step; it is negligible next to an fp16 rounding and next to any sum of ordinary size."""
import math

import numpy as np
import torch

from jnerf_b200.plugin.nerf import IN, N_PARAMS, OUT, W_OFF

ROWS = 128
GB = ROWS * 16                     # bytes of one slab group
S_GROUPS, D_GROUPS = 316, 320
U = 2.0 ** -23                     # per-step error of an fp32 accumulator that truncates
FLOOR = 2.0 ** -12                 # the tensor core's alignment floor, relative to the largest operand (module docstring)

ENC, F, DIR, V = 0, 2112, 2368, 2400
SAVED_COLS, DYS_COLS = 8 * S_GROUPS, 8 * D_GROUPS


def H(l):
    """saved column of h_l, the ReLU output of trunk layer l"""
    return 64 + 256 * l


def DY(l):
    """dys column of kernel layer l's pre-activation gradient"""
    return 256 * l if l < 8 else {8: 2048, 9: 2368, 10: 2496}[l]


def in_cols(l):
    """[(saved column, width)] of kernel layer l's input, concatenated in the weight's column order"""
    if l == 0:
        return [(ENC, 64)]
    if l == 5:
        return [(ENC, 64), (H(4), 256)]
    if l == 9:
        return [(F, 256), (DIR, 32)]
    if l == 10:
        return [(V, 128)]
    return [(H(l - 1), 256)]


# Forward: kernel layer -> [(first weight row, rows, ("saved" | "out", first column), ReLU)]
FWD = {l: [(0, 256, ("saved", H(l)), True)] for l in range(8)}
FWD[8] = [(0, 1, ("out", 3), False), (16, 256, ("saved", F), False)]          # alpha_linear, feature_linear
FWD[9] = [(0, 128, ("saved", V), True)]
FWD[10] = [(0, 3, ("out", 0), False)]

# Dgrad: (kernel layer l, first weight column, columns, saved column of the ReLU mask or None, dys column written), in the kernel's order.
# dY_l (OUT[l] columns at DY(l)) times W_l; layer 9 yields df only (no encoder gradient), layer 5 only its h4 columns.
DGRAD = [(10, 0, 128, V, DY(9)), (9, 0, 256, None, DY(8) + 16), (8, 0, 256, H(7), DY(7))] + \
        [(l, 64 if l == 5 else 0, 256, H(l - 1), DY(l - 1)) for l in range(7, 0, -1)]


def decode(buf, groups, tiles):
    """The first `tiles` blocks of a slab buffer (any dtype; uint8 is read as fp16) -> (tiles * 128, 8 * groups) rows."""
    h = buf.view(torch.float16) if buf.dtype == torch.uint8 else buf
    return h[:tiles * groups * ROWS * 8].view(tiles, groups, ROWS, 8).permute(0, 2, 1, 3).reshape(tiles * ROWS, groups * 8)


def layer_params(P, l):
    """(W (OUT[l], IN[l]), b (OUT[l])) of kernel layer l of the flat vector, float64"""
    W = P[W_OFF[l]:W_OFF[l] + OUT[l] * IN[l]].view(OUT[l], IN[l]).double()
    return W, P[W_OFF[l] + OUT[l] * IN[l]:W_OFF[l + 1]].double()


def layer_input(sv, l):
    return torch.cat([sv[:, c:c + w] for c, w in in_cols(l)], 1)


def pad_mask(device="cpu"):
    """True at the entries of the flat vector that no reference parameter maps to: they must receive exactly zero gradient"""
    m = torch.ones(N_PARAMS, dtype=torch.bool, device=device)
    for l in range(11):
        W = m[W_OFF[l]:W_OFF[l] + OUT[l] * IN[l]].view(OUT[l], IN[l])
        b = m[W_OFF[l] + OUT[l] * IN[l]:W_OFF[l + 1]]
        rows = {8: [0] + list(range(16, 272)), 10: [0, 1, 2]}.get(l, range(OUT[l]))
        cols = {0: range(63), 5: [c for c in range(320) if c != 63], 9: range(283)}.get(l, range(IN[l]))
        W[torch.tensor(list(rows))[:, None], torch.tensor(list(cols))[None, :]] = False
        b[list(rows)] = False
    return m


# ---------------------------------------------------------------------------------------------------------------- exact layers
def _floor(amax, bmax):
    """F of every entry of a product whose entry (i, j) sums over operands of largest magnitudes amax[i] and bmax[j]"""
    return FLOOR * torch.maximum(amax[:, None], bmax[None, :])


def fwd_layer(x, W, b):
    """x W^T + b in float64 and its accumulation bound"""
    x = x.double()
    a = x.abs() @ W.abs().T + b.abs() + _floor(x.abs().amax(1), W.abs().amax(1))
    return x @ W.T + b, (W.shape[1] + 2) * U * a


def dgrad_layer(dy, W):
    """dy W in float64 and its accumulation bound"""
    dy = dy.double()
    return dy @ W, (W.shape[0] + 2) * U * (dy.abs() @ W.abs() + _floor(dy.abs().amax(1), W.abs().amax(0)))


def wgrad_flat(dys, sv):
    """The flat gradient sum_rows dY_l^T X_l (weights) and sum_rows dY_l (biases) of decoded rows, the same sums of magnitudes, and the
    floor F of every weight entry (0 for the biases, which are plain fp32 sums).  Over several row blocks g and a add up, F is the
    largest."""
    g = torch.zeros(N_PARAMS, dtype=torch.float64, device=dys.device)
    a, f = torch.zeros_like(g), torch.zeros_like(g)
    for l in range(11):
        dy, x = dys[:, DY(l):DY(l) + OUT[l]].double(), layer_input(sv, l).double()
        w0, b0 = W_OFF[l], W_OFF[l] + OUT[l] * IN[l]
        g[w0:b0], a[w0:b0] = (dy.T @ x).reshape(-1), (dy.abs().T @ x.abs()).reshape(-1)
        if dy.shape[0]:
            f[w0:b0] = _floor(dy.abs().amax(0), x.abs().amax(0)).reshape(-1)
        g[b0:W_OFF[l + 1]], a[b0:W_OFF[l + 1]] = dy.sum(0), dy.abs().sum(0)
    return g, a, f


def forward_chain(P, enc_pos, enc_dir, rnd=lambda t: t):
    """The whole network from encodings (rows, 64) and (rows, 32) through FWD: (saved (rows, 2528), out (rows, 4)), float64.  rnd is
    applied wherever the kernel stores a value (identity: the exact network)."""
    n = enc_pos.shape[0]
    sv = torch.zeros((n, SAVED_COLS), dtype=torch.float64, device=enc_pos.device)
    out = torch.zeros((n, 4), dtype=torch.float64, device=enc_pos.device)
    sv[:, ENC:ENC + 64], sv[:, DIR:DIR + 32] = enc_pos.double(), enc_dir.double()
    for l in range(11):
        W, b = layer_params(P, l)
        x = layer_input(sv, l)
        for r0, nr, (dst, c), relu in FWD[l]:
            y = fwd_layer(x, W[r0:r0 + nr], b[r0:r0 + nr])[0]
            (sv if dst == "saved" else out)[:, c:c + nr] = rnd(y.clamp_min(0) if relu else y)
    return sv, out


def backward_chain(P, sv, dout, rnd=lambda t: t):
    """dys (rows, 2560) of the dgrad chain through DGRAD from dout (rows, 4), float64, masks read from sv"""
    dys = torch.zeros((sv.shape[0], DYS_COLS), dtype=torch.float64, device=sv.device)
    dys[:, DY(10):DY(10) + 3], dys[:, DY(8)] = dout[:, :3].double(), dout[:, 3].double()
    for l, c0, nc, mask, dst in DGRAD:
        W = layer_params(P, l)[0]
        y = dgrad_layer(dys[:, DY(l):DY(l) + OUT[l]], W[:, c0:c0 + nc])[0]
        if mask is not None:
            y = y * (sv[:, mask:mask + nc] > 0)
        dys[:, dst:dst + nc] = rnd(y)
    return dys


# ---------------------------------------------------------------------------------------------------------------- rounding intervals
def _spacing16(a):
    """gap from fp16 magnitude a (float64, >= 0) to the next larger fp16"""
    e = torch.frexp(a).exponent.to(torch.float64)
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -24), torch.exp2((e - 11).clamp_min(-24)))


def rn16(y):
    """float64 -> the float64 value of the nearest fp16, ties to even, in one rounding (as numpy's float64 -> float16 cast)"""
    a = y.abs()
    q = torch.exp2((torch.frexp(a).exponent.to(torch.float64) - 11).clamp_min(-24))
    r = torch.round(a / q) * q
    return torch.copysign(torch.where(r > 65504, torch.full_like(r, math.inf), r), y)


def ulp32(v):
    """fp32 unit in the last place of |v| (float64)"""
    e = torch.frexp(v.abs()).exponent.to(torch.float64)
    return torch.exp2((e - 24).clamp_min(-149))


def check_rounding(got, y, e, relu=False):
    """(ok, ratio) per entry.  ok: got (fp16) lies in [rn16(y - e), rn16(y + e)], ends clamped at 0 first if relu; compared by value,
    so -0 equals +0.  ratio: the distance from y to the nearest real that rounds to got, over e (0 when y itself rounds to got)."""
    g = got.double()
    lo, hi = y - e, y + e
    if relu:
        lo, hi = lo.clamp_min(0), hi.clamp_min(0)
    ok = (g >= rn16(lo)) & (g <= rn16(hi))
    a = g.abs()
    up, down = _spacing16(a), _spacing16(a * (1 - 2.0 ** -12))
    clo = torch.where(g > 0, g - down / 2, g - up / 2)
    chi = torch.where(g < 0, g + down / 2, g + up / 2)
    if relu:
        clo = torch.where(g == 0, torch.full_like(clo, -math.inf), clo)
    dist = (clo - y).clamp_min(0) + (y - chi).clamp_min(0)
    ratio = torch.where(dist > 0, dist / e, torch.zeros_like(dist))
    return ok, torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)


def freq_encoding(x, L):
    """encode_rows<L> of fp32 coordinates x (rows, 3) in float64: (y, e) over 8-aligned columns [x, sin(x 2^k), cos(x 2^k), ..., 0].
    x 2^k is exact in fp32; sincosf is allowed 2 fp32 ulps of its result; x itself and the padding are exact."""
    x = x.double()
    ys, es = [x], [torch.zeros_like(x)]
    for k in range(L):
        s, c = torch.sin(x * 2.0 ** k), torch.cos(x * 2.0 ** k)
        ys += [s, c]
        es += [2 * ulp32(s), 2 * ulp32(c)]
    w = 3 + 6 * L
    pad = torch.zeros((x.shape[0], (w + 7) // 8 * 8 - w), dtype=torch.float64, device=x.device)
    return torch.cat(ys + [pad], 1), torch.cat(es + [pad], 1)


def numpy_rn16(y):
    """numpy's float64 -> float16 cast, the one-rounding reference rn16 is checked against"""
    with np.errstate(over="ignore"):
        return np.asarray(y, np.float64).astype(np.float16).astype(np.float64)
