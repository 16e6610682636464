"""A float64 reference of the vanilla NeRF network kernels (csrc/nerf_mlp.cu, nerf_mlp.cuh), one layer at a time.

The kernels keep two per-tile slab buffers: `saved`, every layer's input as the forward stored it, and, in the backward's scratch, `dys`,
every layer's pre-activation gradient.  Both are blocks of [groups][128 rows][8 halfs] per 128-row tile.  decode() turns them into
row-major (rows, 8 * groups) matrices whose columns are, at the 8 encoder groups of NeRF and of Mip-NeRF at 8 IPE degrees (Layout
gives the saved columns at the 12 groups of Mip-NeRF at 16 degrees, csrc/mip_mlp_wide.cu):

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

from jnerf_b200.plugin import mip, nerf
from jnerf_b200.plugin.nerf import OUT

ROWS = 128
GB = ROWS * 16                     # bytes of one slab group
D_GROUPS = 320
U = 2.0 ** -23                     # per-step error of an fp32 accumulator that truncates
FLOOR = 2.0 ** -12                 # the tensor core's alignment floor, relative to the largest operand (module docstring)
DYS_COLS = 8 * D_GROUPS


def DY(l):
    """dys column of kernel layer l's pre-activation gradient (the same at every encoder width)"""
    return 256 * l if l < 8 else {8: 2048, 9: 2368, 10: 2496}[l]


class Layout:
    """The column map and parameter layout of the kernels at eg 8-column encoder groups (Layout<EG> of nerf_mlp.cuh).  eg 8: vanilla
    NeRF's 63-column encoding (Mip-NeRF's 48 at 8 IPE degrees uses the same layout); eg 12: Mip-NeRF's 96 columns at 16 IPE degrees,
    which fill the groups.  The saved block puts the encoding first, so every later saved column moves by 8 (eg - 8):

        saved          eg = 8 (316 groups)    eg = 12 (320 groups)
        enc_pos        0 .. 63                0 .. 95
        h_l            64 + 256 l             96 + 256 l
        f              2112 .. 2367           2144 .. 2399
        enc_dir        2368 .. 2399           2400 .. 2431
        v              2400 .. 2527           2432 .. 2559

    The dys block does not depend on eg (module docstring)."""

    def __init__(self, eg):
        E = 8 * eg
        self.eg, self.enc_width = eg, {8: 63, 12: 96}[eg]
        self.ENC, self.F = 0, E + 256 * 8
        self.DIR = self.F + 256
        self.V = self.DIR + 32
        self.S_GROUPS = self.V // 8 + 16
        self.SAVED_COLS = 8 * self.S_GROUPS
        self.IN = mip.kernel_in({8: 8, 12: 16}[eg])
        assert self.IN[0] == E
        self.W_OFF = nerf.w_offsets(self.IN)
        self.N_PARAMS = self.W_OFF[-1]
        # Forward: kernel layer -> [(first weight row, rows, ("saved" | "out", first column), ReLU)]
        self.FWD = {l: [(0, 256, ("saved", self.H(l)), True)] for l in range(8)}
        self.FWD[8] = [(0, 1, ("out", 3), False), (16, 256, ("saved", self.F), False)]          # alpha_linear, feature_linear
        self.FWD[9] = [(0, 128, ("saved", self.V), True)]
        self.FWD[10] = [(0, 3, ("out", 0), False)]
        # Dgrad: (kernel layer l, first weight column, columns, saved column of the ReLU mask or None, dys column written), in the
        # kernel's order.  dY_l (OUT[l] columns at DY(l)) times W_l; layer 9 yields df only (no encoder gradient), layer 5 only its h4
        # columns, which start at 8 eg.
        self.DGRAD = [(10, 0, 128, self.V, DY(9)), (9, 0, 256, None, DY(8) + 16), (8, 0, 256, self.H(7), DY(7))] + \
                     [(l, E if l == 5 else 0, 256, self.H(l - 1), DY(l - 1)) for l in range(7, 0, -1)]

    def H(self, l):
        """saved column of h_l, the ReLU output of trunk layer l"""
        return 8 * self.eg + 256 * l

    def in_cols(self, l):
        """[(saved column, width)] of kernel layer l's input, concatenated in the weight's column order"""
        E = 8 * self.eg
        if l == 0:
            return [(self.ENC, E)]
        if l == 5:
            return [(self.ENC, E), (self.H(4), 256)]
        if l == 9:
            return [(self.F, 256), (self.DIR, 32)]
        if l == 10:
            return [(self.V, 128)]
        return [(self.H(l - 1), 256)]


L8, L12 = Layout(8), Layout(12)

# the 8-group map under its own names (vanilla NeRF, Mip-NeRF at 8 IPE degrees)
S_GROUPS, SAVED_COLS, N_PARAMS, IN, W_OFF = L8.S_GROUPS, L8.SAVED_COLS, L8.N_PARAMS, L8.IN, L8.W_OFF
ENC, F, DIR, V = L8.ENC, L8.F, L8.DIR, L8.V
H, in_cols, FWD, DGRAD = L8.H, L8.in_cols, L8.FWD, L8.DGRAD
assert (IN, W_OFF, N_PARAMS) == (nerf.IN, nerf.W_OFF, nerf.N_PARAMS)


def decode(buf, groups, tiles, t0=0):
    """Blocks t0 .. tiles - 1 of a slab buffer (any dtype; uint8 is read as fp16) -> ((tiles - t0) * 128, 8 * groups) rows."""
    h = buf.view(torch.float16) if buf.dtype == torch.uint8 else buf
    nt = tiles - t0
    return h[t0 * groups * ROWS * 8:tiles * groups * ROWS * 8].view(nt, groups, ROWS, 8).permute(0, 2, 1, 3).reshape(nt * ROWS, groups * 8)


def layer_params(P, l, lay=L8):
    """(W (OUT[l], IN[l]), b (OUT[l])) of kernel layer l of the flat vector, float64"""
    o, i = lay.W_OFF[l], lay.IN[l]
    W = P[o:o + OUT[l] * i].view(OUT[l], i).double()
    return W, P[o + OUT[l] * i:lay.W_OFF[l + 1]].double()


def layer_input(sv, l, lay=L8):
    return torch.cat([sv[:, c:c + w] for c, w in lay.in_cols(l)], 1)


def pad_mask(device="cpu", lay=L8):
    """True at the entries of the flat vector that no reference parameter maps to: they must receive exactly zero gradient"""
    m = torch.ones(lay.N_PARAMS, dtype=torch.bool, device=device)
    E, w = 8 * lay.eg, lay.enc_width
    for l in range(11):
        W = m[lay.W_OFF[l]:lay.W_OFF[l] + OUT[l] * lay.IN[l]].view(OUT[l], lay.IN[l])
        b = m[lay.W_OFF[l] + OUT[l] * lay.IN[l]:lay.W_OFF[l + 1]]
        rows = {8: [0] + list(range(16, 272)), 10: [0, 1, 2]}.get(l, range(OUT[l]))
        cols = {0: range(w), 5: [c for c in range(E + 256) if c < w or c >= E], 9: range(283)}.get(l, range(lay.IN[l]))
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


def wgrad_flat(dys, sv, lay=L8):
    """The flat gradient sum_rows dY_l^T X_l (weights) and sum_rows dY_l (biases) of decoded rows, the same sums of magnitudes, and the
    floor F of every weight entry (0 for the biases, which are plain fp32 sums).  Over several row blocks g and a add up, F is the
    largest."""
    g = torch.zeros(lay.N_PARAMS, dtype=torch.float64, device=dys.device)
    a, f = torch.zeros_like(g), torch.zeros_like(g)
    for l in range(11):
        dy, x = dys[:, DY(l):DY(l) + OUT[l]].double(), layer_input(sv, l, lay).double()
        w0, b0 = lay.W_OFF[l], lay.W_OFF[l] + OUT[l] * lay.IN[l]
        g[w0:b0], a[w0:b0] = (dy.T @ x).reshape(-1), (dy.abs().T @ x.abs()).reshape(-1)
        if dy.shape[0]:
            f[w0:b0] = _floor(dy.abs().amax(0), x.abs().amax(0)).reshape(-1)
        g[b0:lay.W_OFF[l + 1]], a[b0:lay.W_OFF[l + 1]] = dy.sum(0), dy.abs().sum(0)
    return g, a, f


def forward_chain(P, enc_pos, enc_dir, rnd=lambda t: t, lay=L8):
    """The whole network from encodings (rows, 8 eg) and (rows, 32) through FWD: (saved (rows, SAVED_COLS), out (rows, 4)), float64.
    rnd is applied wherever the kernel stores a value (identity: the exact network)."""
    n, E = enc_pos.shape[0], 8 * lay.eg
    sv = torch.zeros((n, lay.SAVED_COLS), dtype=torch.float64, device=enc_pos.device)
    out = torch.zeros((n, 4), dtype=torch.float64, device=enc_pos.device)
    sv[:, lay.ENC:lay.ENC + E], sv[:, lay.DIR:lay.DIR + 32] = enc_pos.double(), enc_dir.double()
    for l in range(11):
        W, b = layer_params(P, l, lay)
        x = layer_input(sv, l, lay)
        for r0, nr, (dst, c), relu in lay.FWD[l]:
            y = fwd_layer(x, W[r0:r0 + nr], b[r0:r0 + nr])[0]
            (sv if dst == "saved" else out)[:, c:c + nr] = rnd(y.clamp_min(0) if relu else y)
    return sv, out


def backward_chain(P, sv, dout, rnd=lambda t: t, lay=L8):
    """dys (rows, 2560) of the dgrad chain through DGRAD from dout (rows, 4), float64, masks read from sv"""
    dys = torch.zeros((sv.shape[0], DYS_COLS), dtype=torch.float64, device=sv.device)
    dys[:, DY(10):DY(10) + 3], dys[:, DY(8)] = dout[:, :3].double(), dout[:, 3].double()
    for l, c0, nc, mask, dst in lay.DGRAD:
        W = layer_params(P, l, lay)[0]
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


def gaussian64(rays, t, ray_shape, integrate):
    """Mip-NeRF's conical (or cylindrical) frustum Gaussians of rays (R, 12) and fenceposts t (R, S + 1) in float64: mean, variance and
    the magnitude |d t_mean| + |o| the fp32 mean is rounded against, (R S, 3) each."""
    rays, t = rays.double(), t.double()
    d, o, r = rays[:, None, 3:6], rays[:, None, 0:3], rays[:, 9:10]
    t0, t1 = t[:, :-1], t[:, 1:]
    if ray_shape == "cone":
        mu, hw = (t0 + t1) / 2, (t1 - t0) / 2
        t_mean = mu + (2 * mu * hw ** 2) / (3 * mu ** 2 + hw ** 2)
        t_var = hw ** 2 / 3 - (4 / 15) * ((hw ** 4 * (12 * mu ** 2 - hw ** 2)) / (3 * mu ** 2 + hw ** 2) ** 2)
        r_var = r ** 2 * (mu ** 2 / 4 + (5 / 12) * hw ** 2 - 4 / 15 * hw ** 4 / (3 * mu ** 2 + hw ** 2))
    else:
        t_mean, r_var, t_var = (t0 + t1) / 2, (r ** 2 / 4).expand_as(t0), (t1 - t0) ** 2 / 12
    mean = d * t_mean[..., None] + o
    d2 = d ** 2
    var = t_var[..., None] * d2 + r_var[..., None] * (1 - d2 / d2.sum(-1, keepdim=True).clamp_min(1e-10))
    if not integrate:
        var = torch.zeros_like(var)
    return mean.reshape(-1, 3), var.reshape(-1, 3), (d.abs() * t_mean[..., None].abs() + o.abs()).reshape(-1, 3)


def ipe64(rays, t, ray_shape="cone", integrate=True, degs=16):
    """The integrated positional encoding in float64, (R S, 6 degs) [sin | cos], degree-major, xyz inner, and the bound of an fp32
    evaluation (mip::ipe).  Column (k, dim): sin / cos(mean 2^k) e^(-var 4^k / 2).  The fp32 mean carries the rounding of mip::gaussian,
    a few ulps of |d t_mean| + |o|, amplified by 2^k; bound: 16 such ulps times 2^k times the attenuation, + 16 ulps of the variance
    term's relative error on the attenuation, + 4 ulps for sincosf / expf and the products."""
    mean, var, mag = gaussian64(rays, t, ray_shape, integrate)
    k = torch.arange(degs, device=mean.device, dtype=torch.float64)
    y = (mean[:, None, :] * 2 ** k[None, :, None]).reshape(-1, 3 * degs)
    vv = (var[:, None, :] * 4 ** k[None, :, None]).reshape(-1, 3 * degs)
    att = torch.exp(-0.5 * vv)
    amp = (mag[:, None, :] * 2 ** k[None, :, None]).reshape(-1, 3 * degs)
    bound = 16 * U * (amp + vv) * att + 4 * U
    return torch.cat([torch.sin(y) * att, torch.cos(y) * att], -1), torch.cat([bound, bound], -1)


def numpy_rn16(y):
    """numpy's float64 -> float16 cast, the one-rounding reference rn16 is checked against"""
    with np.errstate(over="ignore"):
        return np.asarray(y, np.float64).astype(np.float16).astype(np.float64)
