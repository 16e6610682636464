"""The Plenoxels operators of jnerf_b200/ops.py (svox_train_step / svox_render / svox_tv_grad / svox_rmsprop / svox_sample /
svox_weight_render / svox_dilate / svox_compact) restated in plain Python / numpy from the reference's contrib/plenoxel kernels
(volume_render_cuvol_fused.h, render_util.cuh, loss_kernel.h, misc_kernel.h, sample_kernel.h).  Used two ways: as the fp64 reference the
GPU tests compare the kernels against, and installed over jnerf_b200.ops (on top of tests/cpu_backend.py) so that Svox2Runner's host
logic runs without a GPU.  Gradients come back as float arrays; the installed operators convert them to the kernels' fixed point."""
import math

import numpy as np
import torch

FX = 2.0 ** 48
C0, C1 = 0.28209479177387814, 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)


def sh_basis(d):
    x, y, z = d
    return np.array([C0, -C1 * y, C1 * z, -C1 * x, C2[0] * x * y, C2[1] * y * z, C2[2] * (2 * z * z - x * x - y * y), C2[3] * x * z,
                     C2[4] * (x * x - y * y)])


def pixel_ray(c2w, intrin, x, y):
    fx, fy, cx, cy = intrin
    m = np.asarray(c2w, np.float64).reshape(3, 4)
    v = np.array([(x + 0.5 - cx) / fx, (y + 0.5 - cy) / fy, 1.0])
    return m[:, 3].copy(), m[:, :3] @ (v / np.linalg.norm(v))


def find_bounds(o, d, size, xform, step):
    off, scl = np.asarray(xform[:3], np.float64), np.asarray(xform[3:], np.float64)
    o = o * scl + off
    d = d * scl
    ds = 1.0 / np.linalg.norm(d)
    d = d * ds
    tmin, tmax = 0.0, 2e3
    for j in range(3):
        if d[j] != 0:
            t1, t2 = (-0.5 - o[j]) / d[j], (size[j] - 0.5 - o[j]) / d[j]
            tmin, tmax = max(tmin, min(t1, t2)), min(tmax, max(t1, t2))
    return o, d, tmin, tmax, ds * step


def locate(size, o, d, t):
    p, l = np.empty(3), [0, 0, 0]
    for j in range(3):
        x = min(max(o[j] + t * d[j], 0.0), size[j] - 1.0)
        l[j] = min(int(x), size[j] - 2)
        p[j] = x - l[j]
    return l, p


def corner_weights(p):
    w = np.empty(8)
    for k in range(8):
        w[k] = (p[0] if k & 4 else 1 - p[0]) * (p[1] if k & 2 else 1 - p[1]) * (p[2] if k & 1 else 1 - p[2])
    return w


def corner_links(links, l):
    return np.array([links[l[0] + (k >> 2 & 1), l[1] + (k >> 1 & 1), l[2] + (k & 1)] for k in range(8)])


def trace(links, density, sh, xform, opts, o, d, gout=None, grads=None, gout_err=0.0):
    """One ray: rgb (3,); with gout, the gradient of sum(gout * rgb) added into grads = (g_density, g_sh, n_density, n_sh, s_density,
    s_sh): n_* count the terms each entry received, s_* sum each term's scale, the magnitude of the operands its fp32 evaluation
    subtracts or multiplies, with |gout| widened by gout_err (the error of an fp32 dL/drgb) and each weight by the error of its fp32
evaluation.  A density term
    world_step w_k (tc T - accum) has scale world_step w_k (|tc| T + |accum_0| + sum of the |weight tc| subtracted so far): the suffix
    form rounds accum once a sample."""
    step, sigma_thresh, stop_thresh, bg = opts
    size = links.shape
    sph = sh_basis(d)
    o, d, tmin, tmax, ws = find_bounds(o, d, size, xform, step)
    if tmin > tmax:
        return np.full(3, bg)
    sh3 = sh.reshape(-1, 3, 9)
    samples, log_t, out, t = [], 0.0, np.zeros(3), tmin
    while t <= tmax:
        l, p = locate(size, o, d, t)
        lk = corner_links(links, l)
        w = corner_weights(p)
        sigma = sum(w[k] * density[lk[k]] for k in range(8) if lk[k] >= 0)
        if sigma > sigma_thresh:
            coef = sum(w[k] * sh3[lk[k]] for k in range(8) if lk[k] >= 0) if (lk >= 0).any() else np.zeros((3, 9))
            raw = coef @ sph + 0.5
            pcnt = ws * sigma
            t_prev = math.exp(log_t)
            weight = t_prev * (1 - math.exp(-pcnt))
            log_t -= pcnt
            out += weight * np.maximum(raw, 0)
            # the fractional position carries the fp32 error of t d + o, about 4 ulp of (size + t) grid units; a corner weight's scale
            # widens each of its three factors by that error, carried against the bound's 1e-3
            dp = 1e3 * 2.4e-7 * (max(size) + t)
            w_abs = np.array([(p[0] if k & 4 else 1 - p[0]) + dp for k in range(8)]) * \
                np.array([(p[1] if k & 2 else 1 - p[1]) + dp for k in range(8)]) * np.array([(p[2] if k & 1 else 1 - p[2]) + dp for k in range(8)])
            samples.append((lk, w, raw, weight, log_t, t_prev, w_abs))
            if math.exp(log_t) < stop_thresh:
                log_t = -1e3
                break
        t += step
    rgb = out + math.exp(log_t) * bg
    if gout is None:
        return rgb
    gd, gs, nd, ns, sd, ss = grads
    gabs = np.abs(gout) + 1e3 * gout_err          # an absolute error of gout_err, carried against the bound's 1e-3
    accum = float(rgb @ gout)
    scale_a = float(np.abs(rgb) @ gabs)
    for lk, w, raw, weight, lt, t_prev, wk_abs in samples:
        # the kernels' weight T (1 - __expf(-pcnt)) is off by up to ~2 ulp of 1.0 times T (the cancellation in 1 - e^-pcnt): 2.4e-7 T,
        # carried in the scale as 2.4e-4 T against the bound's 1e-3
        w_abs = weight + 2.4e-4 * t_prev
        in01 = (raw >= 0).astype(np.float64)
        tc = float((np.maximum(raw, 0) * gout).sum())
        tc_abs = float((np.maximum(raw, 0) * gabs).sum())
        gcol = (weight * in01 * gout)[:, None] * sph[None, :]
        gcol_abs = (w_abs * in01 * gabs)[:, None] * np.abs(sph)[None, :]
        accum -= weight * tc
        scale_a += w_abs * tc_abs
        gsig = ws * (tc * math.exp(lt) - accum)
        sig_abs = ws * (tc_abs * math.exp(lt) + scale_a)
        for k in range(8):
            if lk[k] >= 0:
                gs[lk[k]] += w[k] * gcol.reshape(27)
                gd[lk[k]] += w[k] * gsig
                ss[lk[k]] += wk_abs[k] * gcol_abs.reshape(27)
                sd[lk[k]] += wk_abs[k] * sig_abs
                ns[lk[k]] += 1
                nd[lk[k]] += 1
    return rgb


def train_step(pix, W, H, c2w, intrin, images, links, density, sh, xform, opts, rgb_err=1e-4):
    """(per-ray squared error (R,), g_density, g_sh, n_density, n_sh, s_density, s_sh) of one step, fp64 (trace() defines n_* and s_*;
    rgb_err bounds the error of an fp32 forward's colour, which enters dL/drgb)."""
    R = len(pix)
    cap = density.shape[0]
    grads = (np.zeros(cap), np.zeros((cap, 27)), np.zeros(cap, np.int64), np.zeros((cap, 27), np.int64), np.zeros(cap), np.zeros((cap, 27)))
    se = np.zeros(R)
    c2w = np.asarray(c2w, np.float64).reshape(-1, 12)
    for i, p in enumerate(np.asarray(pix, np.int64)):
        img, y, x = p // (W * H), (p // W) % H, p % W
        o, d = pixel_ray(c2w[img], intrin, x, y)
        rgb = trace(links, density, sh, xform, opts, o, d)
        px = np.asarray(images[p], np.float64) / 255.0
        gt = px[:3] * px[3] + (1 - px[3])
        se[i] = ((rgb - gt) ** 2).sum()
        trace(links, density, sh, xform, opts, o, d, gout=2 * (rgb - gt) / (3 * R), grads=grads, gout_err=2 * rgb_err / (3 * R))
    return (se,) + grads


def render(n, first, W, c2w, intrin, links, density, sh, xform, opts):
    out = np.zeros((n, 3))
    for i in range(n):
        p = first + i
        o, d = pixel_ray(c2w, intrin, p % W, p // W)
        out[i] = trace(links, density, sh, xform, opts, o, d)
    return out


def tv_grad(links, data, start, n_cells, scale, ignore_edge):
    """tv_grad_sparse_kernel in fp64: the gradient (cap, dim) of the cells (start + i) mod G, i < n_cells."""
    X, Y, Z = links.shape
    data = np.asarray(data, np.float64).reshape(data.shape[0], -1)
    dim = data.shape[1]
    g = np.zeros_like(data)
    flat = links.reshape(-1)
    for i in range(n_cells):
        xyz = (start + i) % (X * Y * Z)
        z, y, x = xyz % Z, xyz // Z % Y, xyz // (Y * Z)
        if ignore_edge and flat[xyz] == 0:
            continue
        l000 = flat[xyz]
        l001 = flat[xyz + 1] if z + 1 < Z else 0
        l010 = flat[xyz + Z] if y + 1 < Y else 0
        l100 = flat[xyz + Y * Z] if x + 1 < X else 0
        v000 = data[l000] if l000 >= 0 else np.zeros(dim)
        nul = v000 if ignore_edge else np.zeros(dim)
        v001 = data[l001] if l001 >= 0 else nul
        v010 = data[l010] if l010 >= 0 else nul
        v100 = data[l100] if l100 >= 0 else nul
        dx, dy, dz = v100 - v000, v010 - v000, v001 - v000
        idelta = scale / np.sqrt(1e-9 + dx * dx + dy * dy + dz * dz)
        dx, dy, dz = dx * (X / 256), dy * (Y / 256), dz * (Z / 256)
        for lk, v in ((l000, -(dx + dy + dz)), (l001, dz), (l010, dy), (l100, dx)):
            if lk >= 0:
                g[lk] += v * idelta
    return g


def rmsprop(p, v, g, lr, alpha, eps):
    """Jittor's RMSprop step on float32 arrays: (p, v) after the step."""
    f = np.float32
    v = f(alpha) * v + (f(1) - f(alpha)) * g * g
    return p - f(lr) * g / (np.sqrt(v) + f(eps)), v


def _fma(a, b, c):
    """fmaf(a, b, c) of float32 arrays: the product of two floats is exact in float64, so one rounding to float64 and one to float32."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _lerp(a, b, w):
    return _fma(w, (b - a).astype(np.float32), a)


def sample(points, links, density, sh, want_sh):
    """sample_grid (grid coordinates) in float32 with the kernels' fmaf lerps: (density (n,), sh (n, 27) or None)."""
    pts = np.asarray(points, np.float32)
    size = np.array(links.shape)
    x = np.minimum(np.maximum(pts, np.float32(0)), (size - 1).astype(np.float32))
    l = np.minimum(x.astype(np.int64), size - 2)
    p = (x - l.astype(np.float32)).astype(np.float32)
    cols = [np.asarray(density, np.float32).reshape(-1, 1)] + ([np.asarray(sh, np.float32)] if want_sh else [])
    data = np.concatenate(cols, 1)
    c = []
    for k in range(8):
        lk = links[l[:, 0] + (k >> 2 & 1), l[:, 1] + (k >> 1 & 1), l[:, 2] + (k & 1)]
        c.append(np.where((lk >= 0)[:, None], data[np.maximum(lk, 0)], np.float32(0)))
    pz, py, px = p[:, 2:3], p[:, 1:2], p[:, 0:1]
    ix0 = _lerp(_lerp(c[0], c[1], pz), _lerp(c[2], c[3], pz), py)
    ix1 = _lerp(_lerp(c[4], c[5], pz), _lerp(c[6], c[7], pz), py)
    v = _lerp(ix0, ix1, px)
    return v[:, 0], (v[:, 1:] if want_sh else None)


def weight_render(data, W, H, c2w, intrin, xform, step, stop_thresh, out):
    """grid_weight_render_kernel in fp64, max-ed into out (X, Y, Z)."""
    fx, fy, cx, cy = intrin
    m = np.asarray(c2w, np.float64).reshape(3, 4)
    size = data.shape
    for iy in range(H):
        for ix in range(W):
            v = np.array([(ix + 0.5 - cx) / fx, (iy + 0.5 - cy) / fy, 1.0])
            o, d, t, tmax, ws = find_bounds(m[:, 3], m[:, :3] @ (v / np.linalg.norm(v)), size, xform, step)
            log_t = 0.0
            while t <= tmax:
                l, p = locate(size, o, d, t)
                w8 = corner_weights(p)
                sigma = sum(w8[k] * data[l[0] + (k >> 2 & 1), l[1] + (k >> 1 & 1), l[2] + (k & 1)] for k in range(8))
                if sigma > 1e-8:
                    att = -ws * sigma
                    w = math.exp(log_t) * (1 - math.exp(att))
                    log_t += att
                    blk = out[l[0]:l[0] + 2, l[1]:l[1] + 2, l[2]:l[2] + 2]
                    np.maximum(blk, w, out=blk)
                    if math.exp(log_t) < stop_thresh:
                        break
                t += step
    return out


def dilate(mask):
    m = np.pad(np.asarray(mask) != 0, 1)
    X, Y, Z = mask.shape
    out = np.zeros((X, Y, Z), bool)
    for i in range(3):
        for j in range(3):
            for k in range(3):
                out |= m[i:i + X, j:j + Y, k:k + Z]
    return out.astype(np.uint8)


def compact(mask, dense, lattice):
    """(links, density, points) of the kept cells, numbered in row-major order."""
    flat = np.asarray(mask).reshape(-1) != 0
    links = np.full(flat.shape, -1, np.int32)
    links[flat] = np.arange(flat.sum(), dtype=np.int32)
    idx = np.nonzero(flat)[0]
    X, Y, Z = mask.shape
    ijk = np.stack([idx // (Y * Z), idx // Z % Y, idx % Z], -1).astype(np.float32)
    lat = np.asarray(lattice, np.float32)
    pts = (lat[:3] + ijk * lat[3:]).astype(np.float32)
    return links.reshape(mask.shape), np.asarray(dense, np.float32).reshape(-1)[flat], pts


def install(monkeypatch, fake=None):
    """cpu_backend.install (unless `fake` is the OracleOps it returned) + the Plenoxels operators, logged in the same call list."""
    import cpu_backend
    if fake is None:
        fake = cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops

    def npy(t):
        return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)

    def to_fx(g):
        return torch.from_numpy(np.rint(np.asarray(g) * FX).astype(np.int64))

    def svox_train_step(pix, W, H, c2w, intrin, images, links, density, sh, xform, opts, grad_density, grad_sh, flag):
        fake._log("svox_train_step")
        se, gd, gs, *_ = train_step(npy(pix), W, H, npy(c2w), intrin, npy(images), npy(links), npy(density).reshape(-1).astype(np.float64),
                                      npy(sh).astype(np.float64), np.asarray(xform, np.float64), opts)
        grad_density += to_fx(gd).view(grad_density.shape)
        grad_sh += to_fx(gs)
        return torch.from_numpy(se.astype(np.float32))

    def svox_render(n, first, W, c2w, intrin, links, density, sh, xform, opts, out=None):
        fake._log("svox_render")
        r = torch.from_numpy(render(n, first, W, npy(c2w), intrin, npy(links), npy(density).reshape(-1).astype(np.float64),
                                    npy(sh).astype(np.float64), np.asarray(xform, np.float64), opts).astype(np.float32))
        if out is None:
            return r
        out.copy_(r)
        return out

    def svox_tv_grad(links, data, start, n_cells, scale, ignore_edge, grad, flag):
        fake._log("svox_tv_grad")
        grad += to_fx(tv_grad(npy(links), npy(data), start, n_cells, scale, ignore_edge)).view(grad.shape)

    def svox_rmsprop(density, sh, grad_density, grad_sh, rms_density, rms_sh, lr_density, lr_sh, alpha_density, alpha_sh, eps):
        fake._log("svox_rmsprop")
        for p, g, v, lr, a in ((density, grad_density, rms_density, lr_density, alpha_density), (sh, grad_sh, rms_sh, lr_sh, alpha_sh)):
            gf = (npy(g).astype(np.float64) / FX).astype(np.float32)
            pn, vn = rmsprop(npy(p), npy(v), gf, lr, a, eps)
            p.copy_(torch.from_numpy(pn))
            v.copy_(torch.from_numpy(vn))
            g.zero_()

    def svox_sample(points, links, density, sh, want_sh):
        fake._log("svox_sample")
        d, s = sample(npy(points), npy(links), npy(density), npy(sh), want_sh)
        return torch.from_numpy(d), (torch.from_numpy(np.ascontiguousarray(s)) if want_sh else None)

    def svox_weight_render(data, W, H, c2w, intrin, xform, step_size, stop_thresh, out):
        fake._log("svox_weight_render")
        o = weight_render(npy(data), W, H, npy(c2w), intrin, np.asarray(xform, np.float64), step_size, stop_thresh, npy(out).astype(np.float64))
        out.copy_(torch.from_numpy(o.astype(np.float32)))
        return out

    def svox_dilate(mask):
        fake._log("svox_dilate")
        return torch.from_numpy(dilate(npy(mask)))

    def svox_compact(mask, dense_density, lattice, capacity):
        fake._log("svox_compact")
        links, d, p = compact(npy(mask), npy(dense_density), lattice)
        assert d.shape[0] == capacity
        return torch.from_numpy(links), torch.from_numpy(d), torch.from_numpy(p)

    for name, fn in (("svox_train_step", svox_train_step), ("svox_render", svox_render), ("svox_tv_grad", svox_tv_grad),
                     ("svox_rmsprop", svox_rmsprop), ("svox_sample", svox_sample), ("svox_weight_render", svox_weight_render),
                     ("svox_dilate", svox_dilate), ("svox_compact", svox_compact)):
        monkeypatch.setattr(real_ops, name, fn)
    return fake


def ref_svox_lib():
    """ctypes handle of oracle/_ref/libref_svox.so (the reference's own Plenoxels kernels, oracle/svox.mk), or None where not built."""
    import ctypes as C
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_svox.so")
    if not os.path.exists(path):
        return None
    lib = C.CDLL(path)
    vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
    lib.ref_svox_render.argtypes = [i32, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.ref_svox_backward.argtypes = [i32, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.ref_svox_tv.argtypes = [i32, vp, vp, i32, i32, i32, vp, i32, i32, f32, i32, vp, vp]
    lib.ref_svox_dilate.argtypes = [i32, i32, i32, vp, vp, vp]
    return lib


def pixel_rays_f32(pix, W, H, c2w, intrin):
    """(origins, unit dirs) (R, 3) float32 of pixel ids, as the rays a JNeRF dataset hands the reference's kernels."""
    c2w = np.asarray(c2w, np.float64).reshape(-1, 12)
    o, d = zip(*(pixel_ray(c2w[p // (W * H)], intrin, p % W, (p // W) % H) for p in np.asarray(pix, np.int64)))
    return np.asarray(o, np.float32), np.asarray(d, np.float32)
