"""Functional wrappers: torch tensors in, C-ABI calls (include/ngp_b200.h) on the current CUDA stream.
torch provides device memory and streams only; every op below runs in libngp_b200.so."""
import numpy as np
import torch

from . import lib

F32, F16 = 0, 1


def _dt(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.float32:
        return F32
    raise TypeError(f"unsupported dtype {t.dtype}")


def _p(t):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "device-resident contiguous tensor required"
    return t.data_ptr()


# The raw handle of torch's current stream.  torch.cuda.current_stream() builds a Stream object and re-checks the device on every call
# (~3 us; 16 calls a training step were a sixth of the step's host time, tools/host_probe.py): the two C getters are what it wraps.
_raw_stream, _raw_device = getattr(torch._C, "_cuda_getCurrentRawStream", None), getattr(torch._C, "_cuda_getDevice", None)


def _stream():
    if _raw_stream is not None and _raw_device is not None:
        return _raw_stream(_raw_device())
    return torch.cuda.current_stream().cuda_stream


class HashLevels:
    """R1: offsets (host, HE/grid_encode.py:17-39) + the device level table the kernels stage in shared memory."""

    def __init__(self, aabb_scale=1, n_levels=16, base_resolution=16, log2_hashmap_size=19, device="cuda", primes=(1, 19349663, 83492791)):
        import ctypes as C
        self.primes = tuple(int(p) & 0xFFFFFFFF for p in primes)
        self.n_levels, self.base_resolution = n_levels, base_resolution
        self.offsets = np.zeros(n_levels + 1, np.uint32)
        pls = C.c_double()
        lib.call("ngp_hash_offsets", float(aabb_scale), n_levels, base_resolution, log2_hashmap_size, self.offsets.ctypes.data, C.addressof(pls))
        self.per_level_scale = pls.value
        self.log2_per_level_scale = float(np.float32(np.log2(self.per_level_scale)))
        self.n_entries = int(self.offsets[-1])
        self.n_params = 2 * self.n_entries
        self.table = torch.empty(n_levels * 32, dtype=torch.uint8, device=device)
        lib.call("ngp_hash_level_table_primes", _stream(), self.offsets.ctypes.data, n_levels, base_resolution, self.log2_per_level_scale,
                 _p(self.table), *self.primes)


def hash_fwd(x, grid, levels):
    out = torch.empty((x.shape[0], 32), dtype=grid.dtype, device=x.device)
    lib.call("ngp_hash_fwd", _stream(), x.shape[0], _p(x), _p(grid), _dt(grid), _p(levels.table), _p(out))
    return out


def hash_bwd(x, dy, levels, grid_grad=None):
    if grid_grad is None:
        # the kernel's memset is skipped for an empty batch (as HE/grid_encode.py:142-144 does): hand out zeros in that case
        alloc = torch.zeros if x.shape[0] == 0 else torch.empty
        grid_grad = alloc(levels.n_params, dtype=dy.dtype, device=x.device)
    lib.call("ngp_hash_bwd", _stream(), x.shape[0], _p(x), _p(dy), _dt(dy), _p(levels.table), _p(grid_grad), levels.n_params)
    return grid_grad


def sh_fwd(dirs, dtype=torch.float16):
    out = torch.empty((dirs.shape[0], 16), dtype=dtype, device=dirs.device)
    lib.call("ngp_sh_fwd", _stream(), dirs.shape[0], _p(dirs), F16 if dtype == torch.float16 else F32, _p(out))
    return out


def mlp_fwd(W, X, n_hidden_matmuls, save_inter=True):
    n = X.shape[0]
    inter = torch.empty(((n_hidden_matmuls + 1) * n, 64), dtype=torch.float16, device=X.device) if save_inter else None
    Y = torch.empty((n, 16), dtype=torch.float16, device=X.device)
    lib.call("ngp_mlp_fwd", _stream(), _p(W), _p(X), _p(inter), _p(Y), n_hidden_matmuls, n)
    return Y, inter


def mlp_bwd(W, X, inter, dY, n_hidden_matmuls, n_out_valid, need_dx=True, need_temps=False):
    n = X.shape[0]
    dX = torch.empty((n, 32), dtype=torch.float16, device=X.device) if need_dx else None
    temps = torch.empty(((n_hidden_matmuls + 1) * n, 64), dtype=torch.float16, device=X.device) if need_temps else None
    dW = torch.empty(W.numel(), dtype=torch.float32, device=X.device)
    lib.call("ngp_mlp_bwd", _stream(), _p(W), _p(X), _p(inter), _p(dY), _p(dX), _p(temps), _p(dW), n_hidden_matmuls, n_out_valid, n)
    return dX, temps, dW


def mlp_bwd_dgrad(W, inter, dY_feature_major, n_hidden_matmuls, need_dx=False):
    """Data-gradient chain only (the contract of the reference's link-level mlp_fused_backward_func): dY is (16, n)."""
    n = dY_feature_major.shape[1]
    dX = torch.empty((n, 32), dtype=torch.float16, device=W.device) if need_dx else None
    temps = torch.empty(((n_hidden_matmuls + 1) * n, 64), dtype=torch.float16, device=W.device)
    lib.call("ngp_mlp_bwd_dgrad", _stream(), _p(W), _p(inter), _p(dY_feature_major), _p(dX), _p(temps), n_hidden_matmuls, n)
    return dX, temps


def network_fwd(coords, grid, levels, wd, wr, n_dev=None, save_enc=True, out=None, enc=None):
    n = coords.shape[0]
    if out is None:
        out = torch.empty((n, 4), dtype=torch.float16, device=coords.device)
    if enc is None and save_enc:
        enc = torch.empty((n, 32), dtype=torch.float16, device=coords.device)
    lib.call("ngp_network_fwd", _stream(), n, _p(n_dev), _p(coords), _p(grid), _p(levels.table), _p(wd), _p(wr), _p(out), _p(enc))
    return out, enc


def network_bwd(coords, enc, levels, wd, wr, dout, grid_grad, dwd, dwr, n_dev=None):
    lib.call("ngp_network_bwd", _stream(), coords.shape[0], _p(n_dev), _p(coords), _p(enc), _p(levels.table), _p(wd), _p(wr), _p(dout),
             _p(grid_grad), _p(dwd), _p(dwr))


_network_bwd = network_bwd        # the Runner folds its optimizer tail into train_sweep only while network_bwd is this function


def network_bwd_scratch(levels, device="cuda"):
    """(fx, w_part): zeroed caller-owned scratch of network_bwd_fx / train_sweep for this level table -- the fixed-point hash-grid
    gradient (int64, two per entry) and the per-CTA weight-gradient slots (fp32)."""
    b = np.zeros(2, np.uint64)
    lib.call("ngp_network_bwd_fx_bytes", levels.n_entries, b.ctypes.data, b[1:].ctypes.data)
    return (torch.zeros(int(b[0]) // 8, dtype=torch.int64, device=device), torch.zeros(int(b[1]) // 4, dtype=torch.float32, device=device))


def network_bwd_fx(coords, enc, levels, wd, wr, dout, fx, w_part, n_dev=None):
    """network_bwd into the scratch of network_bwd_scratch; train_sweep(bwd_rows=coords.shape[0]) turns it into the optimizer step."""
    lib.call("ngp_network_bwd_fx", _stream(), coords.shape[0], _p(n_dev), _p(coords), _p(enc), _p(levels.table), _p(wd), _p(wr), _p(dout),
             levels.n_entries, _p(fx), fx.numel() * fx.element_size(), _p(w_part), w_part.numel() * w_part.element_size())


def train_sweep(table, table_state, fx, w_part, bwd_rows, wd, wd_state, wr, wr_state, lr, step, beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95):
    """The optimizer tail after network_bwd_fx(rows = bwd_rows) in one launch: Adam+EMA of the fp16 hash table and both fp16 MLP weight
    vectors from the backward's scratch, which it clears.  *_state = (m, v, master).  Same bits as network_bwd + three adam_ema calls."""
    assert table.dtype == wd.dtype == wr.dtype == torch.float16 and table.numel() % 2 == 0
    lib.call("ngp_train_sweep", _stream(), table.numel() // 2, _p(table), *map(_p, table_state), _p(fx), _p(w_part), int(bwd_rows), _p(wd),
             *map(_p, wd_state), _p(wr), *map(_p, wr_state), float(lr), float(beta1), float(beta2), float(eps), int(step), float(ema_decay))


def density_fwd(pos, grid, levels, wd):
    out = torch.empty(pos.shape[0], dtype=torch.float16, device=pos.device)
    lib.call("ngp_density_fwd", _stream(), pos.shape[0], _p(pos), _p(grid), _p(levels.table), _p(wd), _p(out))
    return out


# ---- vanilla NeRF (include/ngp_b200.h F1-F4; the parameter layout is plugin/nerf.py's) ----
def nerf_param_count():
    b = np.zeros(1, np.uint64)
    lib.call("ngp_nerf_param_count", b.ctypes.data)
    return int(b[0])


def nerf_workspace_bytes(n):
    """(bytes of the forward's saved activations, bytes of the backward's scratch) for n rows."""
    b = np.zeros(2, np.uint64)
    lib.call("ngp_nerf_workspace_bytes", int(n), b.ctypes.data, b[1:].ctypes.data)
    return int(b[0]), int(b[1])


def nerf_fwd(coords, params, n_dev=None, save=False, out=None):
    """(N,7) NerfCoordinate rows -> ((N,4) fp16 {rgb, alpha}, saved activations for nerf_bwd or None)."""
    n = coords.shape[0]
    if out is None:
        out = torch.empty((n, 4), dtype=torch.float16, device=coords.device)
    saved = torch.empty(max(nerf_workspace_bytes(n)[0], 16), dtype=torch.uint8, device=coords.device) if save else None
    lib.call("ngp_nerf_fwd", _stream(), n, _p(n_dev), _p(coords), _p(params), _p(out), _p(saved))
    return out, saved


def nerf_density(pos, params):
    out = torch.empty(pos.shape[0], dtype=torch.float16, device=pos.device)
    lib.call("ngp_nerf_density", _stream(), pos.shape[0], _p(pos), _p(params), _p(out))
    return out


def nerf_bwd(params, saved, dout, n_dev=None, scratch=None):
    """dout (N,4) fp16 + nerf_fwd's saved activations -> fp32 gradient of the flat parameter vector.  scratch: None, or a caller-owned
    uint8 buffer of at least nerf_workspace_bytes(N)[1] bytes; it then holds every layer's pre-activation gradient and the per-chunk
    weight-gradient partial sums afterwards."""
    n = dout.shape[0]
    need = nerf_workspace_bytes(n)[1]
    if scratch is None:
        scratch = torch.empty(need, dtype=torch.uint8, device=dout.device)
    assert scratch.dtype == torch.uint8 and scratch.numel() >= need, "nerf_bwd: scratch is smaller than nerf_workspace_bytes(N)[1]"
    grad = torch.empty(params.numel(), dtype=torch.float32, device=dout.device)
    lib.call("ngp_nerf_bwd", _stream(), n, _p(n_dev), _p(params), _p(saved), _p(dout), _p(scratch), _p(grad))
    return grad


# ---- Mip-NeRF (include/ngp_b200.h P1-P7; rays (R, 12): origin, direction, viewdir, radius, near, far; t (R, S + 1) fenceposts) ----
RAY_SHAPES = ("cone", "cylinder")


def mip_rays(pix, W, H, c2w, focal, near, far, images):
    """Blender rays of pixel ids pix ((img * H + y) * W + x) -> (rays (n, 12), target rgb (n, 3)).  images: (n_img * H * W, 4) uint8."""
    n = pix.numel()
    rays = torch.empty((n, 12), dtype=torch.float32, device=pix.device)
    target = torch.empty((n, 3), dtype=torch.float32, device=pix.device)
    assert images.dtype == torch.uint8
    lib.call("ngp_mip_rays", _stream(), n, _p(pix), int(W), int(H), _p(c2w), float(focal), float(near), float(far), _p(images), _p(rays), _p(target))
    return rays, target


def mip_sample(rays, n_samples, lindisp, randomized, rng):
    """(R, S + 1) stratified fenceposts; ray g takes the draws [g (S + 1), (g + 1)(S + 1)) of the pcg32 stream `rng` (not advanced here)."""
    t = torch.empty((rays.shape[0], n_samples + 1), dtype=torch.float32, device=rays.device)
    lib.call("ngp_mip_sample", _stream(), rays.shape[0], int(n_samples), _p(rays), int(bool(lindisp)), int(bool(randomized)), int(rng[0]), int(rng[1]), _p(t))
    return t


def mip_resample(t, weights, resample_padding, randomized, rng):
    """(R, S + 1) fenceposts resampled from the blurred weights (R, S); same pcg32 offsets as mip_sample."""
    out = torch.empty_like(t)
    lib.call("ngp_mip_resample", _stream(), t.shape[0], t.shape[1] - 1, _p(t), _p(weights), float(resample_padding), int(bool(randomized)), int(rng[0]),
             int(rng[1]), _p(out))
    return out


def mip_encode(rays, t, ray_shape="cone", integrate=True, min_deg=0):
    """fp32 (IPE (N, 48), view encoding (N, 27)) of the N = R * S intervals, in the reference's column orders."""
    R, S = t.shape[0], t.shape[1] - 1
    enc = torch.empty((R * S, 48), dtype=torch.float32, device=t.device)
    view = torch.empty((R * S, 27), dtype=torch.float32, device=t.device)
    lib.call("ngp_mip_encode", _stream(), R, S, _p(rays), _p(t), RAY_SHAPES.index(ray_shape), int(bool(integrate)), int(min_deg), _p(enc), _p(view))
    return enc, view


def mip_fwd(rays, t, params, ray_shape="cone", integrate=True, min_deg=0, out=None, saved=None):
    """The fused MipNerfMLP forward: (R * S, 4) fp16 {raw rgb, raw density}.  saved: None, or a uint8 buffer of at least
    nerf_workspace_bytes(R * S)[0] bytes for nerf_bwd."""
    R, S = t.shape[0], t.shape[1] - 1
    if out is None:
        out = torch.empty((R * S, 4), dtype=torch.float16, device=t.device)
    lib.call("ngp_mip_fwd", _stream(), R, S, _p(rays), _p(t), RAY_SHAPES.index(ray_shape), int(bool(integrate)), int(min_deg), _p(params), _p(out),
             _p(saved))
    return out


def mip_composite_fwd(raw, t, rays, rgb_padding, density_bias, white_bkgd, weights=True):
    """(rgb (R, 3), acc (R,), distance (R,), weights (R, S) or None)."""
    R, S = t.shape[0], t.shape[1] - 1
    dev = t.device
    rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
    acc = torch.empty(R, dtype=torch.float32, device=dev)
    dist = torch.empty(R, dtype=torch.float32, device=dev)
    w = torch.empty((R, S), dtype=torch.float32, device=dev) if weights else None
    lib.call("ngp_mip_composite_fwd", _stream(), R, S, _p(raw), _dt(raw), _p(t), _p(rays), float(rgb_padding), float(density_bias), int(bool(white_bkgd)),
             _p(rgb), _p(acc), _p(dist), _p(w))
    return rgb, acc, dist, w


def mip_composite_loss_bwd(raw, t, rays, target, mask, rgb_padding, density_bias, white_bkgd, coarse_loss_mult, grad_scale=1.0):
    """Both levels (coarse rows, then fine rows, of the R rays) -> (rgb (2R, 3), per-ray loss terms (2R,), grad_scale * dloss/draw like raw)."""
    R, S = rays.shape[0], t.shape[1] - 1
    assert t.shape[0] == 2 * R and raw.shape[0] == 2 * R * S
    dev = t.device
    rgb = torch.empty((2 * R, 3), dtype=torch.float32, device=dev)
    loss = torch.empty(2 * R, dtype=torch.float32, device=dev)
    draw = torch.empty_like(raw)
    lib.call("ngp_mip_composite_loss_bwd", _stream(), R, S, _p(raw), _dt(raw), _p(t), _p(rays), _p(target), _p(mask), float(rgb_padding), float(density_bias),
             int(bool(white_bkgd)), float(coarse_loss_mult), float(grad_scale), _p(rgb), _p(loss), _p(draw))
    return rgb, loss, draw


# ---- mesh extraction (include/ngp_b200.h M1-M6; tools/extract_mesh.py of the reference) ----
def _mesh_workspace(device, n=0, n_verts=0, n_tris=0):
    b = np.zeros(1, np.uint64)
    lib.call("ngp_mesh_workspace_bytes", int(n), int(n_verts), int(n_tris), b.ctypes.data)
    return torch.empty(max(int(b[0]), 1), dtype=torch.uint8, device=device)


def density_lattice(n, grid, levels, wd):
    """The (n, n, n) fp32 field float(int(max(sigma_raw, 0))) at model positions (i, j, k) / (n-1)."""
    if not 2 <= int(n) <= 1024:
        raise lib.NgpError(f"density_lattice: resolution {n} is outside [2, 1024]")
    field = torch.empty((n, n, n), dtype=torch.float32, device=grid.device)
    lib.call("ngp_density_lattice", _stream(), int(n), _p(grid), _p(levels.table), _p(wd), _p(field))
    return field


def marching_cubes(field, iso=0.5, workspace=None):
    """(n, n, n) fp32 field -> vertices (V, 3) f32 in the PLY frame, triangles (T, 3) int32.  One read-back of the counts per call."""
    import ctypes
    n = field.shape[0]
    assert field.dim() == 3 and field.shape == (n, n, n) and field.dtype == torch.float32
    if workspace is None:
        workspace = _mesh_workspace(field.device, n=n)
    counts = np.zeros(2, np.uint64)
    cp = counts.ctypes.data_as(ctypes.c_void_p)
    lib.call("ngp_marching_cubes", _stream(), n, _p(field), float(iso), _p(workspace), None, 0, None, 0, cp)
    V, T = int(counts[0]), int(counts[1])
    verts = torch.empty((V, 3), dtype=torch.float32, device=field.device)
    tris = torch.empty((T, 3), dtype=torch.int32, device=field.device)
    if T or V:
        lib.call("ngp_marching_cubes", _stream(), n, _p(field), float(iso), _p(workspace), _p(verts), V, _p(tris), T, cp)
    return verts, tris


def mesh_largest_component(verts, tris, workspace=None):
    """The largest edge-connected set of triangles (ties: the one holding the lowest triangle), compacted in order."""
    import ctypes
    V, T = verts.shape[0], tris.shape[0]
    if workspace is None:
        workspace = _mesh_workspace(verts.device, n_verts=V, n_tris=T)
    vo = torch.empty_like(verts)
    to = torch.empty_like(tris)
    counts = np.zeros(2, np.uint64)
    lib.call("ngp_mesh_largest_component", _stream(), V, T, _p(verts), _p(tris), _p(workspace), _p(vo), _p(to), counts.ctypes.data_as(ctypes.c_void_p))
    return vo[:int(counts[0])], to[:int(counts[1])]


def mesh_vertex_normals(verts, tris, workspace=None):
    """Area-weighted unit vertex normals (V, 3) f32, summed in triangle order."""
    V, T = verts.shape[0], tris.shape[0]
    if workspace is None:
        workspace = _mesh_workspace(verts.device, n_verts=V, n_tris=T)
    normals = torch.empty_like(verts)
    lib.call("ngp_mesh_vertex_normals", _stream(), V, T, _p(verts), _p(tris) if T else None, _p(workspace), _p(normals))
    return normals


SMOOTH_METHODS = ("auto", "constrained", "gaussian")


def mesh_smooth_workspace(n, method="auto", device="cuda"):
    b = np.zeros(1, np.uint64)
    lib.call("ngp_mesh_smooth_workspace_bytes", int(n), SMOOTH_METHODS.index(method), b.ctypes.data)
    return torch.empty(int(b[0]), dtype=torch.uint8, device=device)


def mesh_smooth(field, method="auto", max_iters=250, workspace=None):
    """PyMCubes' smooth() of an (n, n, n) fp32 lattice, to be marched at iso 0: "constrained" (signed distance, then a bounded Jacobi
    solve on the band |D| < 4), "gaussian" (sigma 3 of field - 0.5) or "auto" (constrained up to 512^3).  Returns (field_out, info) with
    info = {"method", "iterations", "band_variables"}."""
    n = field.shape[0]
    if method not in SMOOTH_METHODS:
        raise ValueError(f"mesh_smooth: method must be one of {SMOOTH_METHODS}, got {method!r}")
    assert field.dim() == 3 and field.shape == (n, n, n) and field.dtype == torch.float32
    if workspace is None:
        workspace = mesh_smooth_workspace(n, method, field.device)
    out = torch.empty_like(field)
    info = np.zeros(3, np.uint32)
    lib.call("ngp_mesh_smooth", _stream(), n, _p(field), SMOOTH_METHODS.index(method), int(max_iters), _p(workspace), workspace.numel(), _p(out),
             info.ctypes.data)
    return out, dict(method=SMOOTH_METHODS[int(info[0])], iterations=int(info[1]), band_variables=int(info[2]))


# ---- whole-frame renderer with early ray termination (include/ngp_b200.h V1-V4) ----
RENDER_CAPACITY = 1 << 22          # default rows per round: 4 Mi rows = 112 MB of coordinates + 32 MB of network outputs
RENDER_MAX_K = 64


def render_k_steps(capacity, n_alive):
    """Samples per ray of the next round: as many as let every alive ray march in one round, clamp(capacity / n_alive, 1, RENDER_MAX_K).
    Early rounds hold many rays and few samples each (most rays stop or leave the box within a few samples); the last few rays take long
    strides instead of one round per handful of samples.  The output does not depend on this choice."""
    return max(1, min(RENDER_MAX_K, int(capacity) // max(int(n_alive), 1)))


def render_workspace_layout(n_rays, capacity):
    """(bytes, rows offset, network-output offset, row-count offset) of the renderer's workspace."""
    lay = np.zeros(4, np.uint64)
    lib.call("ngp_render_workspace_bytes", int(n_rays), int(capacity), lay.ctypes.data)
    return tuple(int(x) for x in lay)


def render_workspace(n_rays, workspace=None, capacity=RENDER_CAPACITY):
    """`workspace` if it is large enough for n_rays rays at this capacity, else a new one."""
    nbytes = render_workspace_layout(n_rays, capacity)[0]
    if workspace is not None and workspace.numel() >= nbytes:
        return workspace
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")


def render_rays(rays_o, rays_d, bitfield, aabb, cone_angle, near, cascades, const_dt, rng, grid, levels, wd, wr, jitter_tile,
                min_transmittance=0.0, capacity=RENDER_CAPACITY, workspace=None, net=None):
    """Render R rays (model space) to (rgb (R,3) without background, alpha (R,1) = 1 - T, n_samples (R,) int32, rounds).
    Each ray composites the samples ngp_march gives it under the jitter layout of `jitter_tile`-ray tiles, in order, and stops after the
    first sample that brings its transmittance below `min_transmittance` (0: never).  `rng` is not advanced here: the caller moves it
    on by ceil(R / jitter_tile) * 2^32, as the tiled renderer would.  One 4-byte read-back per round.
    net: the network as net(rows, n_dev, out) instead of the fused NGP network of (grid, levels, wd, wr), e.g. OriginNeRFNetworks.infer."""
    import ctypes
    R, dev = rays_o.shape[0], rays_o.device
    nbytes, off_rows, off_net, off_cnt = render_workspace_layout(R, capacity)
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    rows = workspace[off_rows:off_rows + 28 * capacity].view(torch.float32).view(capacity, 7)
    out_rows = workspace[off_net:off_net + 8 * capacity].view(torch.float16).view(capacity, 4)
    n_rows = workspace[off_cnt:off_cnt + 4].view(torch.int32)
    rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
    alpha = torch.empty((R, 1), dtype=torch.float32, device=dev)
    n_samples = torch.empty(R, dtype=torch.int32, device=dev)
    alive = np.zeros(1, np.uint32)
    ap = alive.ctypes.data_as(ctypes.c_void_p)
    lib.call("ngp_render_init", _stream(), R, int(capacity), _p(workspace), float(aabb[0]), float(aabb[1]), _p(rays_o), _p(rays_d), float(cone_angle),
             float(near), int(cascades), int(const_dt), int(rng[0]), int(rng[1]), int(jitter_tile), _p(rgb), _p(alpha), _p(n_samples), ap)
    rounds = 0
    while int(alive[0]):
        n_alive = int(alive[0])
        k = render_k_steps(capacity, n_alive)
        lib.call("ngp_render_march_round", _stream(), R, int(capacity), _p(workspace), n_alive, k, float(aabb[0]), float(aabb[1]), _p(rays_o),
                 _p(rays_d), _p(bitfield), float(cone_angle), int(cascades), int(const_dt))
        bound = min(n_alive, int(capacity) // k) * k                  # rows this round can hold: the network's grid covers no more
        if net is None:
            network_fwd(rows[:bound], grid, levels, wd, wr, n_dev=n_rows, save_enc=False, out=out_rows[:bound])
        else:
            net(rows[:bound], n_rows, out_rows[:bound])
        lib.call("ngp_render_composite_round", _stream(), R, int(capacity), _p(workspace), n_alive, k, float(min_transmittance), int(cascades),
                 _p(rgb), _p(alpha), _p(n_samples), ap)
        rounds += 1
    return rgb, alpha, n_samples, rounds


def march(rays_o, rays_d, bitfield, aabb, max_samples, cone_angle, near, cascades, const_dt, rng, coords=None, workspace=None):
    R = rays_o.shape[0]
    dev = rays_o.device
    counters = torch.empty(2, dtype=torch.int32, device=dev)
    ray_idx = torch.zeros(R, dtype=torch.int32, device=dev)
    numsteps = torch.empty((R, 2), dtype=torch.int32, device=dev)
    if coords is None:
        coords = torch.empty((max_samples, 7), dtype=torch.float32, device=dev)
    if workspace is None:
        workspace = torch.empty(int(lib.load().ngp_march_workspace_bytes(R)), dtype=torch.uint8, device=dev)
    lib.call("ngp_march", _stream(), R, float(aabb[0]), float(aabb[1]), max_samples, _p(rays_o), _p(rays_d), _p(bitfield), float(cone_angle),
             float(near), cascades, int(const_dt), int(rng[0]), int(rng[1]), _p(counters), _p(ray_idx), _p(numsteps), _p(coords), _p(workspace))
    return coords, ray_idx, numsteps, counters


def compact(coords, numsteps, max_compacted, alias=False, zero_fill=True):
    R = numsteps.shape[0]
    dev = coords.device
    out = coords if alias else torch.empty((max_compacted, 7), dtype=torch.float32, device=dev)
    ns = torch.empty((R, 2), dtype=torch.int32, device=dev)
    counters = torch.empty(2, dtype=torch.int32, device=dev)
    lib.call("ngp_compact", _stream(), R, max_compacted, _p(coords), _p(numsteps), _p(out), _p(ns), _p(counters), int(zero_fill))
    return out, ns, counters


def composite_fwd(net, coords, numsteps_in, numsteps_c, bg, cascades=5):
    R = numsteps_c.shape[0]
    rgb = torch.empty((R, 3), dtype=torch.float32, device=net.device)
    lib.call("ngp_composite_fwd", _stream(), R, _p(net), _dt(net), _p(coords), _p(numsteps_in), _p(numsteps_c), _p(bg), cascades, _p(rgb))
    return rgb


def composite_bwd(net, coords, numsteps_c, loss_grad, rgb_ray, mean, cascades=5):
    R = numsteps_c.shape[0]
    dnet = torch.empty_like(net)
    lib.call("ngp_composite_bwd", _stream(), R, net.shape[0], _p(net), _dt(net), _p(coords), _p(numsteps_c), _p(loss_grad), _p(rgb_ray), _p(mean),
             cascades, _p(dnet))
    return dnet


def composite_infer(net, coords, numsteps, cascades=5):
    R = numsteps.shape[0]
    rgb = torch.empty((R, 3), dtype=torch.float32, device=net.device)
    alpha = torch.empty((R, 1), dtype=torch.float32, device=net.device)
    lib.call("ngp_composite_infer", _stream(), R, _p(net), _dt(net), _p(coords), _p(numsteps), cascades, _p(rgb), _p(alpha))
    return rgb, alpha


def composite_loss_bwd(net, coords, numsteps_in, numsteps_c, bg, target, mean, delta=0.1, cascades=5, dnet=None, rgb=None, loss=None, reg_scale=1.0):
    R = numsteps_c.shape[0]
    dev = net.device
    if dnet is None:
        dnet = torch.zeros_like(net)
    if rgb is None:
        rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
    if loss is None:
        loss = torch.empty(R, dtype=torch.float32, device=dev)
    lib.call("ngp_composite_loss_bwd", _stream(), R, net.shape[0], _p(net), _p(coords), _p(numsteps_in), _p(numsteps_c), _p(bg), _p(target),
             float(delta), _p(mean), cascades, _p(rgb), _p(loss), _p(dnet), float(reg_scale))
    return rgb, loss, dnet


def grid_mark_untrained(grid, focal, xforms, res):
    lib.call("ngp_grid_mark_untrained", _stream(), grid.numel(), _p(grid), xforms.shape[0], _p(focal), _p(xforms), int(res[0]), int(res[1]))


def grid_generate_samples(n, rng, step_dev, aabb, grid, n_cascades, thresh):
    pos = torch.empty((n, 3), dtype=torch.float32, device=grid.device)
    idx = torch.empty(n, dtype=torch.int32, device=grid.device)
    lib.call("ngp_grid_generate_samples", _stream(), n, int(rng[0]), int(rng[1]), _p(step_dev), float(aabb[0]), float(aabb[1]), _p(grid), _p(pos),
             _p(idx), n_cascades, float(thresh))
    return pos, idx


def grid_splat(indices, mlp_out, grid_tmp):
    lib.call("ngp_grid_splat", _stream(), indices.numel(), _p(indices), _p(mlp_out), _dt(mlp_out), _p(grid_tmp))


def grid_ema(grid, grid_tmp, decay=0.95):
    lib.call("ngp_grid_ema", _stream(), grid.numel(), float(decay), _p(grid), _p(grid_tmp))


def grid_update_bitfield(grid, mean, bitfield, cascades=5):
    lib.call("ngp_grid_update_bitfield", _stream(), _p(grid), _p(mean), _p(bitfield), cascades)


def adam_ema(param, grad, m, v, master, lr, step, beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95, grad_scale=1.0, zero_grad=True):
    lib.call("ngp_adam_ema", _stream(), param.numel(), _p(param), _dt(param), _p(grad), _dt(grad), float(grad_scale), _p(m), _p(v), _p(master),
             float(lr), float(beta1), float(beta2), float(eps), int(step), float(ema_decay), int(zero_grad))


def raygen(pix, W, H, xforms, focal, principal):
    n = pix.numel()
    dev = pix.device
    img = torch.empty(n, dtype=torch.int32, device=dev)
    o = torch.empty((n, 3), dtype=torch.float32, device=dev)
    d = torch.empty((n, 3), dtype=torch.float32, device=dev)
    lib.call("ngp_raygen", _stream(), n, _p(pix), W, H, _p(xforms), _p(focal), _p(principal), _p(img), _p(o), _p(d))
    return img, o, d


def prepare_batch(pix, W, H, xforms, focal, principal, images, bg):
    n = pix.numel()
    dev = pix.device
    img = torch.empty(n, dtype=torch.int32, device=dev)
    o = torch.empty((n, 3), dtype=torch.float32, device=dev)
    d = torch.empty((n, 3), dtype=torch.float32, device=dev)
    target = torch.empty((n, 3), dtype=torch.float32, device=dev)
    lib.call("ngp_prepare_batch", _stream(), n, _p(pix), W, H, _p(xforms), _p(focal), _p(principal), _p(images), int(images.dtype == torch.uint8),
             _p(bg), _p(img), _p(o), _p(d), _p(target))
    return img, o, d, target


def blend_target(rgba, bg, target=None):
    """target = rgb*a + bg*(1-a) (runner.py:68) for an (n,4) f32 RGBA batch."""
    n = rgba.shape[0]
    if target is None:
        target = torch.empty((n, 3), dtype=torch.float32, device=rgba.device)
    lib.call("ngp_blend_target", _stream(), n, _p(rgba), _p(bg), _p(target))
    return target


def pcg32_seed(seed=1337, seq=1):
    si = np.zeros(2, np.uint64)
    lib.load().ngp_pcg32_seed(seed, seq, si.ctypes.data)
    return si


def pcg32_advance(si, delta=1 << 32):
    lib.load().ngp_pcg32_advance(si.ctypes.data, delta)
    return si


def dp_exchange_step(world, rank, slice_len, n_w, peer_table, peer_table_grad, peer_w_grad, peer_flags, epoch, m, v, master, w_param, w_m, w_v,
                     w_master, lr, step, beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95, grad_scale=1.0):
    """8e: gradient reduce-scatter + Adam/EMA on this rank's table slice + all-gather + MLP-weight all-reduce/update in ONE
    launch over NVLink peer memory.  peer_* are ctypes arrays of `world` device pointers (dp.PeerArena.peers)."""
    import ctypes
    assert m.numel() == slice_len and v.numel() == slice_len and master.numel() == slice_len and w_param.numel() == n_w
    lib.call("ngp_dp_exchange_step", _stream(), int(world), int(rank), int(slice_len), int(n_w), ctypes.addressof(peer_table),
             ctypes.addressof(peer_table_grad), ctypes.addressof(peer_w_grad), ctypes.addressof(peer_flags), int(epoch), _p(m), _p(v), _p(master),
             _p(w_param), _p(w_m), _p(w_v), _p(w_master), float(grad_scale), float(lr), float(beta1), float(beta2), float(eps), int(step),
             float(ema_decay))


def dp_exchange_wait(world, my_flags, epoch):
    lib.call("ngp_dp_exchange_wait", _stream(), int(world), _p(my_flags), int(epoch))


# ---- Plenoxels (include/ngp_b200.h X1-X9; grid = links (X, Y, Z) int32, density (cap,), sh (cap, 27); gradients int64 fixed point) ----
SVOX_FX_UNIT = 2.0 ** -48          # one unit of the fixed-point gradients


def _host_f32(vals):
    a = np.ascontiguousarray(np.asarray(vals, np.float32).reshape(-1))
    return a, a.ctypes.data


def svox_train_step(pix, W, H, c2w, intrin, images, links, density, sh, xform, opts, grad_density, grad_sh, flag):
    """One training step of the rays of pixel ids pix (int32, (img * H + y) * W + x): adds the gradient of the MSE into the int64
    fixed-point grad_density / grad_sh and returns the per-ray squared error (R,).  intrin = (fx, fy, cx, cy); xform = offset[3] +
    scaling[3] (world -> grid); opts = (step_size, sigma_thresh, stop_thresh, background)."""
    R = pix.numel()
    sqerr = torch.empty(R, dtype=torch.float32, device=pix.device)
    xf, xf_p = _host_f32(xform)
    op, op_p = _host_f32(opts)
    X, Y, Z = links.shape
    lib.call("ngp_svox_train_step", _stream(), R, _p(pix), int(W), int(H), _p(c2w), *(float(v) for v in intrin), _p(images), _p(links), X, Y, Z,
             _p(density), _p(sh), xf_p, op_p, _p(grad_density), _p(grad_sh), _p(sqerr), _p(flag))
    return sqerr


def svox_render(n, first, W, c2w, intrin, links, density, sh, xform, opts, out=None):
    """(n, 3) colours of pixels [first, first + n) (row-major) of the camera c2w (12 floats, device)."""
    if out is None:
        out = torch.empty((n, 3), dtype=torch.float32, device=links.device)
    xf, xf_p = _host_f32(xform)
    op, op_p = _host_f32(opts)
    X, Y, Z = links.shape
    lib.call("ngp_svox_render", _stream(), int(n), int(first), int(W), _p(c2w), *(float(v) for v in intrin), _p(links), X, Y, Z, _p(density), _p(sh),
             xf_p, op_p, _p(out))
    return out


def svox_tv_grad(links, data, start, n_cells, scale, ignore_edge, grad, flag):
    """Sparse TV of data (cap, dim) over the cells (start + i) mod (X Y Z), i < n_cells, added into grad (int64 fixed point)."""
    X, Y, Z = links.shape
    dim = data.shape[1] if data.dim() == 2 else 1
    lib.call("ngp_svox_tv_grad", _stream(), _p(links), X, Y, Z, _p(data), dim, int(start), int(n_cells), float(scale), int(bool(ignore_edge)), _p(grad),
             _p(flag))


def svox_rmsprop(density, sh, grad_density, grad_sh, rms_density, rms_sh, lr_density, lr_sh, alpha_density, alpha_sh, eps):
    """RMSprop of both tensors from their fixed-point gradients, which are cleared."""
    lib.call("ngp_svox_rmsprop", _stream(), density.numel(), sh.numel(), _p(density), _p(sh), _p(grad_density), _p(grad_sh), _p(rms_density), _p(rms_sh),
             float(lr_density), float(lr_sh), float(alpha_density), float(alpha_sh), float(eps))


def svox_sample(points, links, density, sh, want_sh):
    """Trilerp at points (n, 3) in grid coordinates -> (density (n,), sh (n, 27) or None)."""
    n = points.shape[0]
    d = torch.empty(n, dtype=torch.float32, device=points.device)
    s = torch.empty((n, 27), dtype=torch.float32, device=points.device) if want_sh else None
    X, Y, Z = links.shape
    lib.call("ngp_svox_sample", _stream(), n, _p(points), _p(links), X, Y, Z, _p(density), _p(sh), int(bool(want_sh)), _p(d), _p(s))
    return d, s


def svox_weight_render(data, W, H, c2w, intrin, xform, step_size, stop_thresh, out):
    """Max-accumulates into out (X, Y, Z) the weights of one camera's rays through the dense density grid data (X, Y, Z)."""
    xf, xf_p = _host_f32(xform)
    X, Y, Z = data.shape
    lib.call("ngp_svox_weight_render", _stream(), int(W), int(H), _p(c2w), *(float(v) for v in intrin), _p(data), X, Y, Z, xf_p, float(step_size),
             float(stop_thresh), _p(out))
    return out


def svox_dilate(mask):
    out = torch.empty_like(mask)
    X, Y, Z = mask.shape
    lib.call("ngp_svox_dilate", _stream(), X, Y, Z, _p(mask), _p(out))
    return out


def svox_compact(mask, dense_density, lattice, capacity):
    """mask (X, Y, Z) uint8 with `capacity` kept cells -> (links (X, Y, Z) int32, density (capacity,), centres (capacity, 3) of the kept
    cells, lattice[0:3] + index * lattice[3:6])."""
    import ctypes as C
    X, Y, Z = mask.shape
    nb = C.c_uint64()
    lib.call("ngp_svox_compact_workspace_bytes", X, Y, Z, C.addressof(nb))
    dev = mask.device
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    links = torch.empty((X, Y, Z), dtype=torch.int32, device=dev)
    dens = torch.empty(capacity, dtype=torch.float32, device=dev)
    pts = torch.empty((capacity, 3), dtype=torch.float32, device=dev)
    lt, lt_p = _host_f32(lattice)
    lib.call("ngp_svox_compact", _stream(), X, Y, Z, _p(mask), _p(dense_density), lt_p, int(capacity), _p(ws), _p(links), _p(dens) if capacity else None,
             _p(pts) if capacity else None)
    return links, dens, pts
