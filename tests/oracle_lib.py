"""ctypes bindings for the oracle (oracle/libngp_oracle.so) and, when present, the host/GPU builds of the
reference's own kernel sources (oracle/_ref/*.so).  TEST INFRASTRUCTURE: imported by tests/, smoke() and the
cpu_baseline / --impl reference legs of bench.py only -- never by the product package."""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")

_u32, _u64, _i64, _f32, _i32 = C.c_uint32, C.c_uint64, C.c_int64, C.c_float, C.c_int
_p = C.c_void_p


def _ptr(a):
    if a is None:
        return None
    assert isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"], "need C-contiguous ndarray"
    return a.ctypes.data_as(C.c_void_p)


def build_oracle():
    so = os.path.join(ORACLE_DIR, "libngp_oracle.so")
    src = os.path.join(ORACLE_DIR, "ngp_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "oracle"])
    return so


_oracle = None


def oracle():
    global _oracle
    if _oracle is None:
        _oracle = C.CDLL(build_oracle())
        _oracle.orc_hash_offsets.restype = C.c_double
        _oracle.orc_hash_offsets.argtypes = [C.c_double, _i32, _i32, _i32, _p]
        _oracle.orc_pcg32_next_float.restype = _f32
        _oracle.orc_grid_mean.restype = _f32
        _oracle.orc_morton3D.restype = _u32
        _oracle.orc_morton3D_invert.restype = _u32
        _oracle.orc_set_level_scales.argtypes = [_p]
        _oracle.orc_set_hash_primes.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        _oracle.orc_set_hash_primes.restype = None
        _oracle.orc_set_reg_scale.argtypes = [C.c_float]
        _oracle.orc_set_reg_scale.restype = None
    return _oracle


def ref(name):
    """Load oracle/_ref/lib<name>.so or return None (the reference tree is absent on the GPU box; the prebuilt
    .so files travel with the snapshot when they were built here)."""
    path = os.path.join(REF_DIR, f"lib{name}.so")
    if not os.path.exists(path):
        return None
    try:
        return C.CDLL(path)
    except OSError:
        return None


# ----------------------------------------------------------------------------------------------------
# hash grid
# ----------------------------------------------------------------------------------------------------
class HashCfg:
    """Level table exactly as HE/grid_encode.py:17-39 computes it."""

    def __init__(self, aabb_scale=1, n_levels=16, base_resolution=16, log2_hashmap_size=19):
        self.n_levels, self.base = n_levels, base_resolution
        self.offsets = np.zeros(n_levels + 1, np.uint32)
        self.per_level_scale = oracle().orc_hash_offsets(float(aabb_scale), n_levels, base_resolution, log2_hashmap_size,
                                                         _ptr(self.offsets))
        self.log2_pls = np.float32(np.log2(self.per_level_scale))  # std::log2(double) narrowed to float arg
        self.n_entries = int(self.offsets[-1])
        self.n_params = self.n_entries * 2


def hash_fwd(cfg, x, grid, acc32=False):
    o = oracle()
    n = x.shape[0]
    x = np.ascontiguousarray(x, np.float32)
    if grid.dtype == np.float32:
        out = np.empty((n, cfg.n_levels * 2), np.float32)
        o.orc_hash_fwd_f32(_u32(n), _ptr(x), _ptr(grid), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base),
                           _f32(cfg.log2_pls), _ptr(out))
    else:
        assert grid.dtype == np.float16
        out = np.empty((n, cfg.n_levels * 2), np.float16)
        fn = o.orc_hash_fwd_f16_acc32 if acc32 else o.orc_hash_fwd_f16
        fn(_u32(n), _ptr(x), _ptr(grid), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(out))
    return out


def hash_indices(cfg, x):
    n = x.shape[0]
    x = np.ascontiguousarray(x, np.float32)
    idx = np.empty((n, cfg.n_levels, 8), np.uint32)
    oracle().orc_hash_indices(_u32(n), _ptr(x), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(idx))
    return idx


def hash_bwd(cfg, x, dy, acc32=False):
    o = oracle()
    n = x.shape[0]
    x = np.ascontiguousarray(x, np.float32)
    dy = np.ascontiguousarray(dy)
    if dy.dtype == np.float32:
        g = np.empty(cfg.n_params, np.float32)
        o.orc_hash_bwd_f32(_u32(n), _ptr(x), _ptr(dy), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(g))
    elif acc32:
        g = np.empty(cfg.n_params, np.float32)
        o.orc_hash_bwd_f16_acc32(_u32(n), _ptr(x), _ptr(dy), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(g))
    else:
        g = np.empty(cfg.n_params, np.float16)
        o.orc_hash_bwd_f16(_u32(n), _ptr(x), _ptr(dy), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(g))
    return g


def hash_bwd_f64(cfg, x, dy):
    """The exact scatter of an fp32 dL/dy (n, 2L): per feature of every entry (g, a, cnt) = (sum dy*w in float64, sum |dy*w|, number of
    nonzero contributions), with the fp32 corner weights w the kernels form."""
    n = x.shape[0]
    x = np.ascontiguousarray(x, np.float32)
    dy = np.ascontiguousarray(dy, np.float32)
    assert dy.shape == (n, cfg.n_levels * 2)
    g = np.empty(cfg.n_params, np.float64)
    a = np.empty(cfg.n_params, np.float64)
    cnt = np.empty(cfg.n_params, np.uint32)
    oracle().orc_hash_bwd_f64(_u32(n), _ptr(x), _ptr(dy), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls),
                              _ptr(g), _ptr(a), _ptr(cnt))
    return g, a, cnt


def ref_hash_fwd(cfg, x, grid):
    r = ref("ref_hash_cpu")
    n = x.shape[0]
    x = np.ascontiguousarray(x, np.float32)
    dt = grid.dtype
    pos_soa = np.empty(3 * n, np.float32)
    enc_soa = np.empty(n * cfg.n_levels * 2, dt)
    out = np.empty((n, cfg.n_levels * 2), dt)
    fn = r.ref_hash_fwd_f32 if dt == np.float32 else r.ref_hash_fwd_f16
    fn(_u32(n), _ptr(x), _ptr(grid), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(pos_soa),
       _ptr(enc_soa), _ptr(out))
    return out, pos_soa


def ref_hash_bwd(cfg, pos_soa, dy):
    r = ref("ref_hash_cpu")
    n = dy.shape[0]
    dt = dy.dtype
    dy = np.ascontiguousarray(dy)
    dy_soa = np.empty(n * cfg.n_levels * 2, dt)
    g = np.empty(cfg.n_params, dt)
    fn = r.ref_hash_bwd_f32 if dt == np.float32 else r.ref_hash_bwd_f16
    fn(_u32(n), _ptr(pos_soa), _ptr(dy), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls), _ptr(dy_soa),
       _ptr(g), _u64(cfg.n_params))
    return g


# ----------------------------------------------------------------------------------------------------
# SH / MLP / network
# ----------------------------------------------------------------------------------------------------
def sh(dirs, dtype=np.float16):
    n = dirs.shape[0]
    dirs = np.ascontiguousarray(dirs, np.float32)
    out = np.empty((n, 16), dtype)
    (oracle().orc_sh_f32 if dtype == np.float32 else oracle().orc_sh_f16)(_u32(n), _ptr(dirs), _ptr(out))
    return out


def mlp_fwd(W, X, n_hidden_matmuls, in_dim=32, width=64, out_pad=16):
    n = X.shape[0]
    W = np.ascontiguousarray(W, np.float16)
    X = np.ascontiguousarray(X, np.float16)
    inter = np.empty(((n_hidden_matmuls + 1) * n, width), np.float16)
    Y = np.empty((n, out_pad), np.float16)
    oracle().orc_mlp_fwd(_u32(n), _u32(in_dim), _u32(width), _u32(out_pad), _u32(n_hidden_matmuls), _ptr(W), _ptr(X), _ptr(inter), _ptr(Y))
    return Y, inter


def mlp_bwd(W, X, inter, dY, n_hidden_matmuls, n_out_valid, in_dim=32, width=64, out_pad=16):
    n = X.shape[0]
    W = np.ascontiguousarray(W, np.float16)
    dX = np.empty((n, in_dim), np.float16)
    temps = np.empty(((n_hidden_matmuls + 1) * n, width), np.float16)
    dW = np.empty(W.shape[0], np.float32)
    oracle().orc_mlp_bwd(_u32(n), _u32(in_dim), _u32(width), _u32(out_pad), _u32(n_hidden_matmuls), _u32(n_out_valid), _ptr(W),
                         _ptr(np.ascontiguousarray(X, np.float16)), _ptr(np.ascontiguousarray(inter, np.float16)),
                         _ptr(np.ascontiguousarray(dY, np.float16)), _ptr(dX), _ptr(temps), _ptr(dW))
    return dX, temps, dW


def network_fwd(cfg, pos, dirs, grid, Wd, Wr, acc32=True):
    n = pos.shape[0]
    out = np.empty((n, 4), np.float16)
    enc = np.empty((n, 32), np.float16)
    h = np.empty((n, 16), np.float16)
    oracle().orc_network_fwd(_u32(n), _ptr(np.ascontiguousarray(pos, np.float32)), _ptr(np.ascontiguousarray(dirs, np.float32)),
                             _ptr(grid), _ptr(cfg.offsets), _u32(cfg.n_levels), _u32(cfg.base), _f32(cfg.log2_pls),
                             _ptr(np.ascontiguousarray(Wd, np.float16)), _ptr(np.ascontiguousarray(Wr, np.float16)), _i32(int(acc32)),
                             _ptr(out), _ptr(enc), _ptr(h))
    return out, enc, h


# ----------------------------------------------------------------------------------------------------
# pcg32
# ----------------------------------------------------------------------------------------------------
def pcg32_seed(seed=1337, seq=1):
    si = np.zeros(2, np.uint64)
    oracle().orc_pcg32_seed(_u64(seed), _u64(seq), _ptr(si))
    return si


def pcg32_advance(si, delta=1 << 32):
    oracle().orc_pcg32_advance(_ptr(si), _i64(delta))
    return si


# ----------------------------------------------------------------------------------------------------
# sampler
# ----------------------------------------------------------------------------------------------------
def march(rays_o, rays_d, bitfield, aabb=(0.0, 1.0), max_samples=4096 * 1024, cone_angle=0.00390625, near=0.2, cascades=5,
          const_dt=True, rng=None):
    R = rays_o.shape[0]
    rng = pcg32_seed() if rng is None else rng
    counters = np.zeros(2, np.uint32)
    ray_idx = np.zeros(R, np.uint32)
    numsteps = np.zeros((R, 2), np.uint32)
    coords = np.zeros((max_samples, 7), np.float32)
    oracle().orc_march(_u32(R), _f32(aabb[0]), _f32(aabb[1]), _u32(max_samples), _ptr(np.ascontiguousarray(rays_o, np.float32)),
                       _ptr(np.ascontiguousarray(rays_d, np.float32)), _ptr(bitfield), _f32(cone_angle), _f32(near), _u32(cascades),
                       _i32(int(const_dt)), _u64(int(rng[0])), _u64(int(rng[1])), _ptr(counters), _ptr(ray_idx), _ptr(numsteps), _ptr(coords))
    return coords, ray_idx, numsteps, counters


def ref_march(rays_o, rays_d, bitfield, aabb=(0.0, 1.0), max_samples=4096 * 1024, cone_angle=0.00390625, near=0.2, const_dt=True,
              rng=None, n_images=1):
    sfx = "constdt" if const_dt else "cone"
    r = ref(f"ref_sampler_cpu_{sfx}")
    R = rays_o.shape[0]
    rng = pcg32_seed() if rng is None else rng
    counters = np.zeros(2, np.uint32)
    ray_idx = np.zeros(R, np.uint32)
    numsteps = np.zeros((R, 2), np.uint32)
    coords = np.zeros((max_samples, 7), np.float32)
    metadata = np.zeros((n_images, 11), np.float32)
    metadata[:, 4:6] = 0.5
    metadata[:, 6:8] = 1000.0
    imgs = np.zeros(R, np.uint32)
    xforms = np.zeros((n_images, 12), np.float32)
    getattr(r, f"ref_march_{sfx}")(_u32(R), _f32(aabb[0]), _f32(aabb[1]), _u32(max_samples), _ptr(np.ascontiguousarray(rays_o, np.float32)),
                                   _ptr(np.ascontiguousarray(rays_d, np.float32)), _ptr(bitfield), _f32(cone_angle), _ptr(metadata),
                                   _ptr(imgs), _ptr(counters), _ptr(ray_idx), _ptr(numsteps), _ptr(coords), _ptr(xforms), _f32(near),
                                   _u64(int(rng[0])), _u64(int(rng[1])))
    return coords, ray_idx, numsteps, counters


def compact(coords, numsteps, max_compacted):
    R = numsteps.shape[0]
    out = np.zeros((max_compacted, 7), np.float32)
    ns_out = np.zeros((R, 2), np.uint32)
    counters = np.zeros(2, np.uint32)
    oracle().orc_compact(_u32(R), _u32(max_compacted), _ptr(coords), _ptr(numsteps), _ptr(out), _ptr(ns_out), _ptr(counters))
    return out, ns_out, counters


def ref_compact(coords, numsteps, max_compacted, net_out=None):
    r = ref("ref_sampler_cpu_constdt")
    R = numsteps.shape[0]
    out = np.zeros((max_compacted, 7), np.float32)
    ns_out = np.zeros((R, 2), np.uint32)
    c_steps, c_rays = np.zeros(1, np.uint32), np.zeros(1, np.uint32)
    if net_out is None:
        net_out = np.zeros((coords.shape[0], 4), np.float32)
    r.ref_compact_constdt(_u32(R), _f32(0), _f32(1), _u32(max_compacted), _ptr(np.ascontiguousarray(net_out, np.float32)), _ptr(coords),
                          _ptr(out), _ptr(numsteps), _ptr(c_steps), _ptr(ns_out), _ptr(c_rays))
    return out, ns_out, np.array([c_steps[0], c_rays[0]], np.uint32)


def composite_fwd(net, coords, numsteps_in, numsteps_c, bg, cascades=5):
    R = numsteps_c.shape[0]
    rgb = np.empty((R, 3), np.float32)
    net = np.ascontiguousarray(net)
    oracle().orc_composite_fwd(_u32(R), _ptr(net), _i32(int(net.dtype == np.float16)), _ptr(coords), _ptr(numsteps_in), _ptr(numsteps_c),
                               _ptr(np.ascontiguousarray(bg, np.float32)), _u32(cascades), _ptr(rgb))
    return rgb


def composite_infer(net, coords, numsteps, cascades=5):
    R = numsteps.shape[0]
    rgb = np.empty((R, 3), np.float32)
    alpha = np.empty((R, 1), np.float32)
    net = np.ascontiguousarray(net)
    oracle().orc_composite_infer(_u32(R), _ptr(net), _i32(int(net.dtype == np.float16)), _ptr(coords), _ptr(numsteps), _u32(cascades),
                                 _ptr(rgb), _ptr(alpha))
    return rgb, alpha


def composite_bwd(net, coords, numsteps_c, loss_grad, rgb_ray, mean, cascades=5):
    R = numsteps_c.shape[0]
    net = np.ascontiguousarray(net)
    dnet = np.empty_like(net)
    oracle().orc_composite_bwd(_u32(R), _u32(net.shape[0]), _ptr(net), _i32(int(net.dtype == np.float16)), _ptr(coords), _ptr(numsteps_c),
                               _ptr(np.ascontiguousarray(loss_grad, np.float32)), _ptr(np.ascontiguousarray(rgb_ray, np.float32)),
                               _f32(mean), _u32(cascades), _ptr(dnet))
    return dnet


def composite_f64(net, coords, numsteps_in, numsteps_c, bg, cascades=5, loss_scale=None, l1=0.0, loss_grad=None, rgb_ray=None):
    """The composite in float64 with per-entry error bounds for an fp32 evaluation (orc_composite_f64).  numsteps_in None: inference
    (no background).  loss_grad / rgb_ray None: forward only.  loss_scale defaults to the kernels' fp32 128 / R.  Returns a dict of
    rgb, rgb_err (R,3), T, T_err, alpha, alpha_err (R,) and, for the backward, dnet, dnet_err (N,4), NaN where no ray covers a row."""
    R = numsteps_c.shape[0]
    net = np.ascontiguousarray(net)
    N = net.shape[0]
    if loss_scale is None:
        loss_scale = np.float32(128) / np.float32(R)
    out = {k: np.zeros((R, 3)) for k in ("rgb", "rgb_err")}
    out.update({k: np.zeros(R) for k in ("T", "T_err", "alpha", "alpha_err")})
    bwd = loss_grad is not None
    out["dnet"] = np.full((N, 4), np.nan) if bwd else None
    out["dnet_err"] = np.full((N, 4), np.nan) if bwd else None
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    u32 = lambda a: None if a is None else np.ascontiguousarray(a).view(np.uint32)
    args = [f32(coords), u32(numsteps_in), u32(numsteps_c), f32(bg), f32(loss_grad), f32(rgb_ray)]      # alive until the call returns
    co, ns_in, ns_c, bg_, lg, rr = (_ptr(a) for a in args)
    oracle().orc_composite_f64(_u32(R), _ptr(net), _i32(int(net.dtype == np.float16)), co, ns_in, ns_c, bg_, _u32(cascades), _f32(loss_scale),
                               _f32(l1), lg, rr, _ptr(out["rgb"]), _ptr(out["rgb_err"]), _ptr(out["T"]), _ptr(out["T_err"]),
                               _ptr(out["alpha"]), _ptr(out["alpha_err"]), _ptr(out["dnet"]), _ptr(out["dnet_err"]))
    return out


def ref_composite(net, coords, numsteps_in, numsteps_c, bg, loss_grad=None, mean=0.0):
    r = ref("ref_sampler_cpu_constdt")
    R = numsteps_c.shape[0]
    net = np.ascontiguousarray(net)
    t = "f16" if net.dtype == np.float16 else "f32"
    rgb = np.empty((R, 3), np.float32)
    getattr(r, f"ref_rgb_fwd_{t}_constdt")(_u32(R), _f32(0), _f32(1), _ptr(net), _ptr(coords), _ptr(numsteps_in), _ptr(rgb), _ptr(numsteps_c),
                                           _ptr(np.ascontiguousarray(bg, np.float32)))
    dnet = None
    if loss_grad is not None:
        dnet = np.empty_like(net)
        m = np.array([mean], np.float32)
        getattr(r, f"ref_rgb_bwd_{t}_constdt")(_u32(R), _u32(net.shape[0]), _f32(0), _f32(1), _ptr(dnet), _ptr(net), _ptr(numsteps_c), _ptr(coords),
                                               _ptr(np.ascontiguousarray(loss_grad, np.float32)), _ptr(rgb), _ptr(m))
    rgb_i = np.empty((R, 3), np.float32)
    alpha = np.empty((R, 1), np.float32)
    bg3 = np.zeros(3, np.float32)
    getattr(r, f"ref_rgb_infer_{t}_constdt")(_u32(R), _f32(0), _f32(1), _ptr(bg3), _ptr(net), _ptr(coords), _ptr(numsteps_c), _ptr(rgb_i), _ptr(alpha))
    return rgb, dnet, rgb_i, alpha


def huber_grad(x, target, delta=0.1):
    x = np.ascontiguousarray(x, np.float32).ravel()
    t = np.ascontiguousarray(target, np.float32).ravel()
    g = np.empty_like(x)
    l = np.empty_like(x)
    oracle().orc_huber_grad(_u32(x.size), _ptr(x), _ptr(t), _f32(delta), _ptr(g), _ptr(l))
    return g, l


# ----------------------------------------------------------------------------------------------------
# occupancy grid
# ----------------------------------------------------------------------------------------------------
G3 = 128 ** 3


def mark_untrained(grid, focal, xforms, res):
    n_img = xforms.shape[0]
    oracle().orc_mark_untrained(_u32(grid.size), _ptr(grid), _u32(n_img), _ptr(np.ascontiguousarray(focal, np.float32)),
                                _ptr(np.ascontiguousarray(xforms, np.float32)), _i32(res[0]), _i32(res[1]))
    return grid


def generate_grid_samples(n, rng, step, aabb, grid, n_cascades, thresh):
    pos = np.empty((n, 3), np.float32)
    idx = np.empty(n, np.uint32)
    oracle().orc_generate_grid_samples(_u32(n), _u64(int(rng[0])), _u64(int(rng[1])), _u32(step), _f32(aabb[0]), _f32(aabb[1]), _ptr(grid),
                                       _ptr(pos), _ptr(idx), _u32(n_cascades), _f32(thresh))
    return pos, idx


def splat(indices, mlp_out, grid_tmp):
    mlp_out = np.ascontiguousarray(mlp_out)
    oracle().orc_splat(_u32(indices.size), _ptr(indices), _ptr(mlp_out), _i32(int(mlp_out.dtype == np.float16)), _ptr(grid_tmp))
    return grid_tmp


def ema(grid, grid_tmp, decay=0.95):
    oracle().orc_ema(_u32(grid.size), _f32(decay), _ptr(grid), _ptr(grid_tmp))
    return grid


def grid_mean(grid):
    return float(oracle().orc_grid_mean(_ptr(grid)))


def update_bitfield(grid, mean, cascades=5):
    bits = np.zeros(G3 * 5 // 8, np.uint8)
    oracle().orc_update_bitfield(_ptr(grid), _f32(mean), _u32(cascades), _ptr(bits))
    return bits


def adam_ema(param, grad, m, v, master, lr, step, b1=0.9, b2=0.99, eps=1e-15, decay=0.95):
    oracle().orc_adam_ema(_u64(param.size), _ptr(param), _i32(int(param.dtype == np.float16)), _ptr(grad), _ptr(m), _ptr(v), _ptr(master),
                          _f32(lr), _f32(b1), _f32(b2), _f32(eps), _u32(step), _f32(decay))


def raygen(pix, W, H, xforms, focal, principal):
    n = pix.size
    img = np.empty(n, np.uint32)
    o = np.empty((n, 3), np.float32)
    d = np.empty((n, 3), np.float32)
    oracle().orc_raygen(_u32(n), _ptr(np.ascontiguousarray(pix, np.uint32)), _u32(W), _u32(H), _ptr(np.ascontiguousarray(xforms, np.float32)),
                        _ptr(np.ascontiguousarray(focal, np.float32)), _ptr(np.ascontiguousarray(principal, np.float32)), _ptr(img), _ptr(o), _ptr(d))
    return img, o, d


# ----------------------------------------------------------------------------------------------------
# synthetic scene helpers shared by tests / bench (not reference semantics)
# ----------------------------------------------------------------------------------------------------
def sphere_bitfield(radius=0.3, center=(0.5, 0.5, 0.5), cascades=5, shell=None):
    """Occupancy bitfield of an analytic solid sphere (or, with `shell`, a spherical shell of that half-thickness) in the
    unit cube, built through the oracle's grid path."""
    grid = np.zeros(G3 * 5, np.float32)
    ids = np.arange(G3, dtype=np.uint32)
    def minv(x):
        x = x & 0x49249249
        x = (x | (x >> 2)) & 0xc30c30c3
        x = (x | (x >> 4)) & 0x0f00f00f
        x = (x | (x >> 8)) & 0xff0000ff
        x = (x | (x >> 16)) & 0x0000ffff
        return x
    x, y, z = minv(ids), minv(ids >> 1), minv(ids >> 2)
    for lvl in range(cascades):
        sc = 2.0 ** lvl
        px = ((x + 0.5) / 128 - 0.5) * sc + 0.5
        py = ((y + 0.5) / 128 - 0.5) * sc + 0.5
        pz = ((z + 0.5) / 128 - 0.5) * sc + 0.5
        d2 = (px - center[0]) ** 2 + (py - center[1]) ** 2 + (pz - center[2]) ** 2
        inside = d2 < radius * radius if shell is None else np.abs(np.sqrt(d2) - radius) < shell
        grid[lvl * G3:(lvl + 1) * G3] = np.where(inside, 1.0, 0.0)
    return update_bitfield(grid, 1.0, cascades), grid


def random_rays(R, seed=0, radius=1.3):
    """Cameras on a sphere around the unit-cube centre looking roughly at it."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(R, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    o = 0.5 + radius * v
    tgt = 0.5 + rng.uniform(-0.35, 0.35, size=(R, 3))
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)
