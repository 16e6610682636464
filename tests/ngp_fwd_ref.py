"""Float64 references of the fused NGP network (csrc/fused_net.cu): the mirror of its forward and backward, a rigorous per-entry interval
for its forward outputs, the degree-4 SH features with an fp32 evaluation bound, and the routing-probe weight sets.

The forward chain, with an fp16 rounding wherever the kernel stores to a shared-memory slab:

    enc (32) -> relu(W0d .) -> hd (64) -> Woutd . -> h (16; h0 is the density output) -> rin = [h | SH] (32) -> relu(W0r .) -> h1 (64)
             -> relu(W1r .) -> h2 (64) -> Woutr[:3] . -> rgb

Interval.  Each value is carried as a centre x, the float64 mirror that rounds to fp16 where the kernel does, and a radius E that bounds
how far the kernel's fp16 value can be from x.  For a layer z = W x the kernel sums the products of its own inputs, which lie within E of
x, so its fp32 sum lies within |W| E + acc of z, acc = (K + 2) 2^-23 (|W| (|x| + E) + F) being the accumulation bound of nerf_mlp_ref
(F is the tensor core's alignment floor, measured there).  ReLU and rn16 are monotone, so the stored value lies in
[lo16, hi16] = [rn16(relu(z - |W| E - acc)), rn16(relu(z + |W| E + acc))], and the next layer's radius is E' = max(hi16 - x', x' - lo16)
with x' = rn16(relu(z)).  The encoding enters with E = 0 (the kernel's own, checked bit for bit against the oracle).  The interval is
rigorous but loose after a few layers: one possible flip in any of 64 hidden units widens every downstream entry.  A rounding-mode slip
therefore stays inside it; agreement with the mirror, tile by tile, is what catches that.

SH.  sh4 (ngp_common.cuh; SphericalEncode.h) in float64 from the fp32 direction, with a bound on any fp32 evaluation of the same
expressions, contracted to FMA or not.  It is a running error bound: every fp32 quantity q is a float64 value v and a bound e on
|fp32 q - v|.  A rounding adds u (|v| + e) + eta, u = 2^-24 and eta = 2^-150 (half the smallest fp32 subnormal); so
- x = 2 dx - 1 (and y, z): 2 dx is exact, one rounding: e_x = u |x| + eta;
- a constant c (an fp32 literal of the float64 one): e_c = u |c|; 1, 3 and 5 are exact;
- a product ab: |a| e_b + |b| e_a + e_a e_b, then a rounding -- x y, x z, y z, x^2, y^2, z^2, every c t and the products of o[9..15];
- a sum a + b: e_a + e_b, then a rounding.  These are the differences that cancel: o[6] = c z^2 - d, o[8] = c x^2 - c y^2,
  o[9] (-3 x^2 + y^2), o[11] and o[13] (1 - 5 z^2), o[12] (5 z^2 - 3), o[14] (x^2 - y^2) and o[15] (-x^2 + 3 y^2).  Their bound is
  absolute, so it does not blow up where the result is near zero.
A fused multiply-add skips the product's rounding; the bound grows with every input bound, so the unfused bound covers it.  The fp16
feature lies in [rn16(v - e), rn16(v + e)].

The kernel's SH is not the oracle's bit for bit.  nvcc contracts seven of the sixteen terms to FMA in the fused kernels (o[6], o[8],
o[9], o[11], o[12], o[13], o[15], read from the SASS), while the oracle evaluates them unfused (-ffp-contract=off).  Both are correct fp32
evaluations and lie in the interval above, but about one fp16 feature in 12 000 rounds the other way.  sh_f32() reproduces either
evaluation exactly (a correctly rounded fp32 FMA is emulated in float64), and the GPU tests hold the kernel's routed SH to the
contracted one bit for bit."""
import numpy as np
import torch

from nerf_mlp_ref import _spacing16, check_rounding, fwd_layer, rn16

ROWS = 128
WD_N, WR_N = 64 * 32 + 16 * 64, 64 * 32 + 64 * 64 + 16 * 64


def _h(x):
    """One fp16 rounding, where the kernel stores a value to a slab."""
    return x.to(torch.float16).to(torch.float64)


def split_weights(wd, wr):
    """(W0d, Woutd, W0r, W1r, Woutr) of the flat fp16 weight vectors, float64, on their device"""
    wd, wr = wd.to(torch.float64), wr.to(torch.float64)
    return wd[:2048].view(64, 32), wd[2048:].view(16, 64), wr[:2048].view(64, 32), wr[2048:6144].view(64, 64), wr[6144:].view(16, 64)


def mirror(enc, sh, dout, wd, wr):
    """The fused network's forward and backward in float64 from fp16 tensors enc (n,32), sh (n,16), dout (n,4), wd, wr (flat), on their
    device.  Returns out (n,4), the slab values, d_enc, and per weight vector (dwd, dwr) the gradient and the sum of |term|."""
    f = lambda t: t.to(torch.float64)
    W0d, Woutd, W0r, W1r, Woutr = split_weights(wd, wr)
    enc, dout = f(enc), f(dout)
    hd = _h(torch.relu(enc @ W0d.T))
    h = _h(hd @ Woutd.T)
    rin = torch.cat([h, f(sh)], 1)
    h1 = _h(torch.relu(rin @ W0r.T))
    h2 = _h(torch.relu(h1 @ W1r.T))
    out = torch.cat([_h(h2 @ Woutr[:3].T), h[:, :1]], 1)
    dYr = dout[:, :3]
    g_h2 = _h((dYr @ Woutr[:3]) * (h2 > 0))
    g_h1 = _h((g_h2 @ W1r) * (h1 > 0))
    dYd = g_h1 @ W0r[:, :16]
    dYd[:, 0] += dout[:, 3]                                  # dL/dsigma joins before the one rounding, as the kernel adds it in fp32
    dYd = _h(dYd)
    g_hd = _h((dYd @ Woutd) * (hd > 0))
    d_enc = _h(g_hd @ W0d)
    pairs_d = [(g_hd, enc), (dYd, hd)]                       # W0d [out][in] = g_hd^T enc, Woutd [out][in] = dYd^T hd
    pairs_r = [(g_h1, rin), (g_h2, h1), (dYr, h2)]           # W0r, W1r, Woutr (rows >= 3 zero)

    def grads(pairs, n_w):
        g, a = torch.zeros(n_w, dtype=torch.float64, device=enc.device), torch.zeros(n_w, dtype=torch.float64, device=enc.device)
        o = 0
        for x, y in pairs:
            gx, ax = (x.T @ y).reshape(-1), (x.abs().T @ y.abs()).reshape(-1)
            g[o:o + gx.numel()], a[o:o + gx.numel()] = gx, ax
            o += gx.numel() if x.shape[1] != 3 else 16 * 64
        assert o == n_w
        return g, a

    slabs = dict(hd=hd, h=h, rin=rin, h1=h1, h2=h2, g_h2=g_h2, g_h1=g_h1, dYd=dYd, g_hd=g_hd, d_enc_abs=g_hd.abs() @ W0d.abs())
    return out, slabs, d_enc, grads(pairs_d, WD_N), grads(pairs_r, WR_N)


# ---------------------------------------------------------------------------------------------------------------- SH
C0, C1, C4, C6A, C6B = 0.28209479177387814, 0.48860251190291987, 1.0925484305920792, 0.94617469575755997, 0.31539156525251999
C8, C9, C10, C11, C12, C14 = 0.54627421529603959, 0.59004358992664352, 2.8906114426405538, 0.45704579946446572, 0.3731763325901154, 1.4453057213202769
U24, ETA = 2.0 ** -24, 2.0 ** -150


def sh_f64(dirs):
    """(v, e) (n, 16) float64 of fp32 directions (n, 3) (a numpy array or a tensor): the exact basis and the fp32 evaluation bound of
    the module docstring."""
    d = torch.as_tensor(np.asarray(dirs, np.float32) if not torch.is_tensor(dirs) else dirs).to(torch.float64)

    def rnd(v, e):
        return v, e + U24 * (v.abs() + e) + ETA

    def mul(a, b):
        return rnd(a[0] * b[0], a[0].abs() * b[1] + b[0].abs() * a[1] + a[1] * b[1])

    def add(a, b):
        return rnd(a[0] + b[0], a[1] + b[1])

    def const(c):
        return torch.full_like(d[:, 0], c), torch.full_like(d[:, 0], U24 * abs(c))

    def exact(c):
        return torch.full_like(d[:, 0], c), torch.zeros_like(d[:, 0])

    def neg(a):
        return -a[0], a[1]

    x, y, z = (rnd(2 * d[:, i] - 1, torch.zeros_like(d[:, i])) for i in range(3))
    xy, xz, yz, x2, y2, z2 = mul(x, y), mul(x, z), mul(y, z), mul(x, x), mul(y, y), mul(z, z)
    z5 = mul(exact(5.0), z2)
    o = [const(C0), mul(const(-C1), y), mul(const(C1), z), mul(const(-C1), x), mul(const(C4), xy), mul(const(-C4), yz),
         add(mul(const(C6A), z2), const(-C6B)), mul(const(-C4), xz), add(mul(const(C8), x2), neg(mul(const(C8), y2))),
         mul(mul(const(C9), y), add(mul(exact(-3.0), x2), y2)), mul(mul(const(C10), xy), z),
         mul(mul(const(C11), y), add(exact(1.0), neg(z5))), mul(mul(const(C12), z), add(z5, exact(-3.0))),
         mul(mul(const(C11), x), add(exact(1.0), neg(z5))), mul(mul(const(C14), z), add(x2, neg(y2))),
         mul(mul(const(C9), x), add(neg(x2), mul(exact(3.0), y2)))]
    return torch.stack([t[0] for t in o], 1), torch.stack([t[1] for t in o], 1)


def sh_interval(dirs):
    """[lo16, hi16] (n, 16) float64: the fp16 values any fp32 evaluation of sh4 can store"""
    v, e = sh_f64(dirs)
    return rn16(v - e), rn16(v + e)


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c) of float32 arrays: the product is exact in float64, the sum is rounded once to float64 and its
    error recovered (TwoSum); only where that float64 sum is an fp32 rounding tie does the error decide the direction."""
    a, b, c = (np.asarray(t, np.float32).astype(np.float64) for t in np.broadcast_arrays(a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    t = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    nb = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (s != r64) & (s == (r64 + nb.astype(np.float64)) / 2) & (t != 0)
    return np.where(tie, np.where(t > 0, np.maximum(r, nb), np.minimum(r, nb)), r).astype(np.float32)


def sh_f32(dirs, contract=True):
    """sh4 of fp32 directions (n, 3) in fp32, term by term as compiled: contract=True as the fused kernels' SASS evaluates it (seven
    terms contracted to FMA), contract=False as the oracle's C (-ffp-contract=off).  Returns (n, 16) float32."""
    d = np.asarray(dirs, np.float32)
    f = np.float32
    mul = lambda a, b: (np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)).astype(np.float32)
    add = lambda a, b: fma32(a, f(1), b)
    mad = (lambda a, b, c: fma32(a, b, c)) if contract else (lambda a, b, c: add(mul(a, b), c))
    x, y, z = (fma32(d[:, i], f(2), f(-1)) for i in range(3))
    xy, xz, yz, x2, y2, z2 = mul(x, y), mul(x, z), mul(y, z), mul(x, x), mul(y, y), mul(z, z)
    c = lambda v: f(v)
    o = [np.full_like(x, c(C0)), mul(c(-C1), y), mul(c(C1), z), mul(c(-C1), x), mul(c(C4), xy), mul(c(-C4), yz),
         mad(z2, c(C6A), c(-C6B)), mul(c(-C4), xz),
         mad(x2, c(C8), -mul(y2, c(C8))) if contract else add(mul(c(C8), x2), -mul(c(C8), y2)),
         mul(mul(c(C9), y), mad(x2, f(-3), y2)), mul(mul(xy, c(C10)), z),
         mul(mul(c(C11), y), mad(z2, f(-5), f(1))), mul(mul(c(C12), z), mad(z2, f(5), f(-3))),
         mul(mul(c(C11), x), mad(z2, f(-5), f(1))), mul(mul(c(C14), z), add(x2, -y2)),
         mul(mul(c(C9), x), mad(y2, f(3), -x2))]
    return np.stack(o, 1)


# ---------------------------------------------------------------------------------------------------------------- interval chain
def _layer(x, E, W, relu):
    """(x', lo16, hi16, E', z, r) of one layer z = W x on centres x and radii E (module docstring): the kernel's fp32 sum lies within r
    of z, its stored value in [lo16, hi16]"""
    z = x @ W.T
    _, acc = fwd_layer(x.abs() + E, W, torch.zeros(W.shape[0], dtype=torch.float64, device=x.device))
    r = E @ W.abs().T + acc
    lo, hi, zr = z - r, z + r, z
    if relu:
        zr, lo, hi = z.clamp_min(0), lo.clamp_min(0), hi.clamp_min(0)
    x1, lo16, hi16 = rn16(zr), rn16(lo), rn16(hi)
    return x1, lo16, hi16, torch.maximum(hi16 - x1, x1 - lo16), z, r


def interval_chain(enc, sh, sh_lo, sh_hi, wd, wr):
    """The forward from the kernel's encoding enc (n, 32) and the SH centre sh (n, 16) with its interval [sh_lo, sh_hi], all on one
    device.  Returns dict: out (n, 4) the mirror's outputs, lo / hi (n, 4) their intervals, z / r (n, 4) the exact sums and their radii
    before the rounding, the radii E of hd, h, SH, h1, h2, and hidden: per hidden layer (x, lo16, hi16)."""
    W0d, Woutd, W0r, W1r, Woutr = split_weights(wd, wr)
    enc, sh, sh_lo, sh_hi = (t.to(torch.float64) for t in (enc, sh, sh_lo, sh_hi))
    hd, hd_lo, hd_hi, E_hd, _, _ = _layer(enc, torch.zeros_like(enc), W0d, True)
    h, h_lo, h_hi, E_h, h_z, h_r = _layer(hd, E_hd, Woutd, False)
    E_sh = torch.maximum(sh_hi - sh, sh - sh_lo)
    h1, h1_lo, h1_hi, E_h1, _, _ = _layer(torch.cat([h, sh], 1), torch.cat([E_h, E_sh], 1), W0r, True)
    h2, h2_lo, h2_hi, E_h2, _, _ = _layer(h1, E_h1, W1r, True)
    rgb, lo, hi, _, z, r = _layer(h2, E_h2, Woutr[:3], False)
    cat = lambda a, b: torch.cat([a, b[:, :1]], 1)
    return dict(out=cat(rgb, h), lo=cat(lo, h_lo), hi=cat(hi, h_hi), z=cat(z, h_z), r=cat(r, h_r),
                E=dict(hd=E_hd, h=E_h, sh=E_sh, h1=E_h1, h2=E_h2),
                hidden=dict(hd=(hd, hd_lo, hd_hi), h=(h, h_lo, h_hi), h1=(h1, h1_lo, h1_hi), h2=(h2, h2_lo, h2_hi)))


def interval_check(got, ch):
    """(inside (n, 4) bool, ratio (n, 4)) of the kernel's outputs got against the chain's intervals (check_rounding of nerf_mlp_ref:
    ratio is the distance from the exact centre z to the nearest real that rounds to got, over the radius r; inside <=> ratio <= 1)."""
    return check_rounding(got, ch["z"], ch["r"])


def radius_ulps(ch):
    """the output radii max(hi16 - x, x - lo16) in fp16 ulps of the centre x, (n, 4)"""
    x = ch["out"]
    return torch.maximum(ch["hi"] - x, x - ch["lo"]) / _spacing16(x.abs())


def tile_agreement(got, centre, min_rows=64):
    """(n_tiles_held, 4): per 128-row tile with at least min_rows rows, the share of each output column equal to the mirror.  Rows are
    the live rows from row 0."""
    eq = (got.to(torch.float64) == centre).to(torch.float64)
    n = eq.shape[0]
    full = n // ROWS
    shares = [eq[:full * ROWS].view(full, ROWS, 4).mean(1)]
    if n - full * ROWS >= min_rows:
        shares.append(eq[full * ROWS:].mean(0, keepdim=True))
    return torch.cat(shares, 0)


# ---------------------------------------------------------------------------------------------------------------- routing probes
def probe_sets():
    """The probe weight sets as [(k0, [src_0, src_1, src_2])]: out[:, 3] = h0 = enc[:, k0], and colour channel i reads rin column c_i,
    src_i = (c_i, k_i) with h_{c_i} = enc[:, k_i] for c_i < 16, or (c_i, None) for the SH feature c_i - 16.  Eight sets route each of the 32
    encoded features and each of h1..h15 to an output column at least once, six more each of the 16 SH features."""
    sets = []
    for r in range(8):
        sets.append((r, [(1 + (3 * r + i) % 15, 8 + 3 * r + i) for i in range(3)]))
    for r in range(6):
        sets.append((8 + r, [(16 + (3 * r + i) % 16, None) for i in range(3)]))
    return sets


def probe_weights(k0, srcs):
    """Flat fp16 (wd, wr) of one probe set.  W0d = [I32; -I32] gives hd = [relu(enc) | relu(-enc)]; Woutd row j = e_k - e_{32+k} gives
    h_j = enc_k; W0r rows 2i, 2i+1 = +-e_{c_i}, W1r the identity on rows 0..5 and Woutr row i = e_{2i} - e_{2i+1} give rgb_i = rin_{c_i}.
    Every product is an fp16 value times +-1 and every sum has one nonzero term, so each output is exactly the routed input."""
    w0d = np.zeros((64, 32), np.float16)
    w0d[np.arange(32), np.arange(32)] = 1
    w0d[32 + np.arange(32), np.arange(32)] = -1
    woutd = np.zeros((16, 64), np.float16)
    woutd[0, k0], woutd[0, 32 + k0] = 1, -1
    w0r, w1r, woutr = np.zeros((64, 32), np.float16), np.zeros((64, 64), np.float16), np.zeros((16, 64), np.float16)
    for i, (c, k) in enumerate(srcs):
        if k is not None:
            woutd[c] = 0
            woutd[c, k], woutd[c, 32 + k] = 1, -1
        w0r[2 * i, c], w0r[2 * i + 1, c] = 1, -1
        w1r[2 * i, 2 * i] = w1r[2 * i + 1, 2 * i + 1] = 1
        woutr[i, 2 * i], woutr[i, 2 * i + 1] = 1, -1
    return np.concatenate([w0d.ravel(), woutd.ravel()]), np.concatenate([w0r.ravel(), w1r.ravel(), woutr.ravel()])


def probe_expected(k0, srcs, enc, sh16):
    """(n, 4) fp16 values the probe set must produce exactly, from the encoding enc (n, 32) and the SH features sh16 (n, 16)"""
    cols = [enc[:, k] if k is not None else sh16[:, c - 16] for c, k in srcs] + [enc[:, k0]]
    return torch.stack([torch.as_tensor(c) for c in cols], 1)
