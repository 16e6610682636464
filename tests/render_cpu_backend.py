"""The whole-frame renderer of jnerf_b200/ops.py (render_rays) on CPU tensors, installed on top of tests/cpu_backend.py so that the host
logic of Runner.render_rays / render_img_with_pose / render / test runs without a GPU.  Test infrastructure, like cpu_backend.

The stand-in is built only from pieces that are pinned against the reference elsewhere: the oracle's march, one call per jitter tile
with one rng.advance() between tiles; the oracle's network on the marched rows; and a sequential numpy composite per ray, in sample
order, with the stopping rule (a ray stops after the first sample that brings T below min_transmittance)."""
import numpy as np
import torch

import cpu_backend
import oracle_lib as ol

MIN_CONE = np.float32(1.73205080757 / 1024.0)


def _np(t, dtype=None):
    a = t.detach().cpu().numpy()
    return np.ascontiguousarray(a if dtype is None else a.astype(dtype, copy=False))


def composite_sequential(net, dt_warped, counts, cascades, min_transmittance):
    """Per ray (rows [base, base + count) in ray order): w = alpha T, rgb += w c, T *= 1 - alpha, sample by sample, stopping after the
    first sample with T < min_transmittance.  float32 throughout.  Returns rgb (R,3), alpha (R,1), n_samples (R,)."""
    R = counts.shape[0]
    base = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    o = net.astype(np.float32)
    c = (1.0 / (1.0 + np.exp(-o[:, :3]))).astype(np.float32)
    mx = np.float32(MIN_CONE * (1 << (cascades - 1)))
    dt = (dt_warped.astype(np.float32) * (mx - MIN_CONE) + MIN_CONE).astype(np.float32)
    a = (1.0 - np.exp(-np.exp(o[:, 3]) * dt)).astype(np.float32)
    rgb = np.zeros((R, 3), np.float32)
    T = np.ones(R, np.float32)
    n = np.zeros(R, np.int32)
    live = counts > 0
    for s in range(int(counts.max()) if R else 0):
        idx = np.nonzero(live & (s < counts))[0]
        if idx.size == 0:
            break
        row = base[idx] + s
        w = (a[row] * T[idx]).astype(np.float32)
        rgb[idx] = (rgb[idx] + w[:, None] * c[row]).astype(np.float32)
        T[idx] = (T[idx] * (np.float32(1) - a[row])).astype(np.float32)
        n[idx] += 1
        live[idx[T[idx] < np.float32(min_transmittance)]] = False
    return rgb, (1 - T)[:, None].astype(np.float32), n


def install(monkeypatch, fake=None):
    """cpu_backend.install (unless `fake` is the OracleOps it returned) + render_rays / render_workspace, logged in the same call list."""
    if fake is None:
        fake = cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops

    def render_workspace(n_rays, workspace=None, capacity=real_ops.RENDER_CAPACITY):
        return workspace

    def render_rays(rays_o, rays_d, bitfield, aabb, cone_angle, near, cascades, const_dt, rng, grid, levels, wd, wr, jitter_tile,
                    min_transmittance=0.0, capacity=real_ops.RENDER_CAPACITY, workspace=None):
        fake._log("render_rays")
        if int(capacity) <= 0 or int(jitter_tile) <= 0:
            raise RuntimeError("render_rays: capacity and jitter_tile must be positive")
        R, tile = rays_o.shape[0], int(jitter_tile)
        o_all, d_all, bits = _np(rays_o, np.float32), _np(rays_d, np.float32), _np(bitfield, np.uint8)
        st = np.array([int(rng[0]), int(rng[1])], np.uint64)
        rgb, alpha, n = np.zeros((R, 3), np.float32), np.zeros((R, 1), np.float32), np.zeros(R, np.int32)
        for p in range(0, R, tile):
            o, d = o_all[p:p + tile], d_all[p:p + tile]
            coords, _, numsteps, counters = ol.march(o, d, bits, aabb, tile * 1024, cone_angle, near, cascades, const_dt, st)
            ol.pcg32_advance(st)
            total = int(counters[1])
            counts = numsteps[:, 0].astype(np.int64)
            if total:
                c = coords[:total]
                net, _, _ = ol.network_fwd(levels.cfg, c[:, :3].copy(), c[:, 4:].copy(), _np(grid), _np(wd, np.float16),
                                           _np(wr, np.float16), acc32=True)
                rgb[p:p + tile], alpha[p:p + tile], n[p:p + tile] = composite_sequential(net, c[:, 3], counts, cascades, min_transmittance)
        rounds = 1 if R else 0
        return torch.from_numpy(rgb), torch.from_numpy(alpha), torch.from_numpy(n), rounds

    monkeypatch.setattr(real_ops, "render_rays", render_rays)
    monkeypatch.setattr(real_ops, "render_workspace", render_workspace)
    return fake
