"""The Mip-NeRF operators of jnerf_b200/ops.py (mip_rays / mip_sample / mip_resample / mip_encode / mip_composite_fwd /
mip_composite_loss_bwd) restated from the reference's numpy / Jittor code (contrib/mipnerf utils/miputils.py, dataset/nerf_datasets.py) in
torch, with the kernels' pcg32 uniforms restated on the host.  Used two ways: installed over jnerf_b200.ops (on top of tests/cpu_backend.py)
so that MipRunner's host logic runs without a GPU, and as the fp64 reference the GPU tests compare the kernels against."""
import math

import numpy as np
import torch

_M = 0x5851F42D4C957F2D


def pcg32_uniforms(rng, n_rays, per_ray):
    """(n_rays, per_ray) float64: draw j of ray g is draw g * per_ray + j of the pcg32 stream at rng = (state, inc), as next_float()."""
    state, inc = int(rng[0]), int(rng[1])

    def advance(st, delta):
        cur_mult, cur_plus, acc_mult, acc_plus = _M, inc, 1, 0
        while delta > 0:
            if delta & 1:
                acc_mult = acc_mult * cur_mult % 2 ** 64
                acc_plus = (acc_plus * cur_mult + cur_plus) % 2 ** 64
            cur_plus = (cur_mult + 1) * cur_plus % 2 ** 64
            cur_mult = cur_mult * cur_mult % 2 ** 64
            delta //= 2
        return (acc_mult * st + acc_plus) % 2 ** 64

    s = np.array([advance(state, g * per_ray) for g in range(n_rays)], np.uint64)
    out = np.empty((n_rays, per_ray), np.float64)
    with np.errstate(over="ignore"):
        for j in range(per_ray):
            old = s
            s = old * np.uint64(_M) + np.uint64(inc)
            xs = (((old >> np.uint64(18)) ^ old) >> np.uint64(27)).astype(np.uint32)
            rot = (old >> np.uint64(59)).astype(np.uint32)
            u = (xs >> rot) | (xs << ((-rot.astype(np.int64)) & 31).astype(np.uint32))
            out[:, j] = ((u >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32).astype(np.float64) - 1.0
    return out


def blender_rays_numpy(c2w, focal, W, H, near, far):
    """nerf_datasets.py:193-235 for every pixel of each camera, in the reference's fp32 numpy (radius: the float64 division by sqrt(12)
    rounded to fp32) -> (n_img * H * W, 12) float32 rows."""
    x, y = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing="xy")
    f = np.float32(focal)
    cam = np.stack([(x - np.float32(W * 0.5) + np.float32(0.5)) / f, -((y - np.float32(H * 0.5) + np.float32(0.5)) / f), -np.ones_like(x)], -1)
    rows = []
    for m in np.asarray(c2w, np.float32).reshape(-1, 3, 4):
        R = m[:3, :3]
        d = cam[..., 0:1] * R[:, 0] + cam[..., 1:2] * R[:, 1] + cam[..., 2:3] * R[:, 2]       # camera_dirs @ R^T, term by term
        o = np.broadcast_to(m[:3, 3], d.shape)
        v = d / np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])[..., None]
        e = d[:-1] - d[1:]
        dx = np.sqrt((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2])
        dx = np.concatenate([dx, dx[-2:-1]], 0)
        radii = ((dx * np.float32(2)).astype(np.float64) / np.sqrt(12)).astype(np.float32)[..., None]
        ones = np.ones_like(radii)
        rows.append(np.concatenate([o, d, v, radii, ones * np.float32(near), ones * np.float32(far)], -1).reshape(-1, 12))
    return np.concatenate(rows, 0)


def sample(rays, S, lindisp, randomized, u=None):
    """sample_along_rays (:324-362); u (R, S + 1) the uniforms."""
    near, far = rays[:, 10:11], rays[:, 11:12]
    v = torch.linspace(0.0, 1.0, S + 1, dtype=rays.dtype, device=rays.device)
    t = 1.0 / (1.0 / near * (1.0 - v) + 1.0 / far * v) if lindisp else near + (far - near) * v
    if randomized:
        mids = 0.5 * (t[:, 1:] + t[:, :-1])
        upper = torch.cat([mids, t[:, -1:]], -1)
        lower = torch.cat([t[:, :1], mids], -1)
        t = lower + (upper - lower) * u
    return t


def resample(t, w, padding, randomized, u=None):
    """resample_along_rays + sorted_piecewise_constant_pdf (:61-117, :365-408); u (R, S + 1) the uniforms (randomized)."""
    eps32 = float(np.finfo(np.float32).eps)
    wp = torch.cat([w[:, :1], w, w[:, -1:]], -1)
    wm = torch.maximum(wp[:, :-1], wp[:, 1:])
    w = 0.5 * (wm[:, :-1] + wm[:, 1:]) + padding
    ws = w.sum(-1, keepdim=True)
    pad = torch.clamp(1e-5 - ws, min=0)
    w = w + pad / w.shape[-1]
    ws = ws + pad
    cdf = torch.clamp(torch.cumsum((w / ws)[:, :-1], -1), max=1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf, torch.ones_like(cdf[:, :1])], -1)
    n = t.shape[-1]
    if randomized:
        s = 1.0 / n
        u = torch.clamp(torch.arange(n, dtype=t.dtype, device=t.device) * s + (s - eps32) * u, max=1 - eps32)
    else:
        u = torch.linspace(0.0, 1 - eps32, n, dtype=t.dtype, device=t.device).expand(t.shape[0], n)
    mask = u[:, None, :] >= cdf[:, :, None]

    def find(x):
        x0 = torch.where(mask, x[:, :, None], x[:, :1, None]).max(-2).values
        x1 = torch.where(~mask, x[:, :, None], x[:, -1:, None]).min(-2).values
        return x0, x1
    b0, b1 = find(t)
    c0, c1 = find(cdf)
    f = torch.clamp(torch.nan_to_num((u - c0) / (c1 - c0), 0.0), 0, 1)
    return b0 + f * (b1 - b0)


def encode(rays, t, ray_shape="cone", integrate=True, min_deg=0, max_deg=8):
    """cast_rays + integrated_pos_enc (:138-275) -> (N, 48) and pos_enc(viewdir, 0, 4) (:120-127) -> (N, 27), rows ray-major."""
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
    cov = t_var[..., None] * d2 + r_var[..., None] * (1 - d2 / torch.clamp(d2.sum(-1, keepdim=True), min=1e-10))
    if not integrate:
        cov = torch.zeros_like(cov)
    scales = torch.tensor([2.0 ** i for i in range(min_deg, max_deg)], dtype=t.dtype, device=t.device)
    y = (mean[..., None, :] * scales[:, None]).reshape(mean.shape[:-1] + (-1,))
    yv = (cov[..., None, :] * scales[:, None] ** 2).reshape(mean.shape[:-1] + (-1,))
    enc = torch.exp(-0.5 * torch.cat([yv, yv], -1)) * torch.sin(torch.cat([y, y + 0.5 * math.pi], -1))
    x = rays[:, 6:9]
    xb = (x[:, None, :] * torch.tensor([1.0, 2.0, 4.0, 8.0], dtype=t.dtype, device=t.device)[:, None]).reshape(-1, 12)
    view = torch.cat([x, torch.sin(torch.cat([xb, xb + 0.5 * math.pi], -1))], -1)
    S = t.shape[1] - 1
    return enc.reshape(-1, 48), view.repeat_interleave(S, 0)


def composite(raw, t, rays, p, bias, white):
    """rays2rgb + volumetric_rendering (:83-96, :278-321): (rgb, distance, acc, weights); raw (R * S, 4), differentiable."""
    R, S = t.shape[0], t.shape[1] - 1
    raw = raw.reshape(R, S, 4)
    rgb = torch.sigmoid(raw[..., :3]) * (1 + 2 * p) - p
    density = torch.nn.functional.softplus(raw[..., 3] + bias)
    t_mids = 0.5 * (t[:, :-1] + t[:, 1:])
    delta = (t[:, 1:] - t[:, :-1]) * rays[:, None, 3:6].norm(dim=-1)
    sd = density * delta
    alpha = 1 - torch.exp(-sd)
    trans = torch.exp(-torch.cat([torch.zeros_like(sd[:, :1]), torch.cumsum(sd[:, :-1], -1)], -1))
    w = alpha * trans
    comp = (w[..., None] * rgb).sum(-2)
    acc = w.sum(-1)
    dist = torch.where(acc > 0, (w * t_mids).sum(-1) / acc, t[:, 0])           # the kernels' t_0 for 0 / 0
    dist = torch.minimum(torch.maximum(dist, t[:, 0]), t[:, -1])
    if white:
        comp = comp + (1 - acc[:, None])
    return comp, dist, acc, w


def loss_and_grad(raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale=1.0):
    """runner.py:83-92 over both levels (coarse rows first) and its gradient with respect to raw, by autograd: (rgb (2R,3), per-ray loss
    terms (2R,), grad_scale * dloss/draw)."""
    R = rays.shape[0]
    raw = raw.detach().clone().requires_grad_()
    rays2 = torch.cat([rays, rays])
    with torch.enable_grad():
        rgb = composite(raw, t, rays2, p, bias, white)[0]
        m = torch.ones(R, dtype=raw.dtype, device=raw.device) if mask is None else mask.to(raw.dtype)
        mult = torch.cat([torch.full((R,), coarse_mult, dtype=raw.dtype, device=raw.device), torch.ones(R, dtype=raw.dtype, device=raw.device)])
        per_ray = mult * torch.cat([m, m]) * ((rgb - torch.cat([target, target])) ** 2).sum(-1) / m.sum()
        (per_ray.sum() * grad_scale).backward()
    return rgb.detach(), per_ray.detach(), raw.grad


def install(monkeypatch, fake=None):
    """cpu_backend.install (unless `fake` is the OracleOps it returned) + the Mip-NeRF operators in fp32, logged in the same call list."""
    import cpu_backend
    if fake is None:
        fake = cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops

    def mip_rays(pix, W, H, c2w, focal, near, far, images):
        fake._log("mip_rays")
        all_rays = torch.from_numpy(blender_rays_numpy(c2w.cpu().numpy(), focal, W, H, near, far))
        idx = pix.long()
        return all_rays[idx], images[idx, :3].float() / 255.0

    def _u(rng, R, S):
        return torch.from_numpy(pcg32_uniforms(rng, R, S + 1)).float()

    def mip_sample(rays, S, lindisp, randomized, rng):
        fake._log("mip_sample")
        return sample(rays, S, lindisp, randomized, _u(rng, rays.shape[0], S) if randomized else None)

    def mip_resample(t, weights, padding, randomized, rng):
        fake._log("mip_resample")
        return resample(t, weights, padding, randomized, _u(rng, t.shape[0], t.shape[1] - 1) if randomized else None)

    def mip_encode(rays, t, ray_shape="cone", integrate=True, min_deg=0):
        fake._log("mip_encode")
        return encode(rays, t, ray_shape, integrate, min_deg, min_deg + 8)

    def mip_composite_fwd(raw, t, rays, p, bias, white, weights=True):
        fake._log("mip_composite_fwd")
        rgb, dist, acc, w = composite(raw.float(), t, rays, p, bias, white)
        return rgb, acc, dist, (w if weights else None)

    def mip_composite_loss_bwd(raw, t, rays, target, mask, p, bias, white, coarse_mult, grad_scale=1.0):
        fake._log("mip_composite_loss_bwd")
        rgb, loss, g = loss_and_grad(raw.float(), t, rays, target, mask, p, bias, white, coarse_mult, grad_scale)
        return rgb, loss, g.to(raw.dtype)

    for name, fn in (("mip_rays", mip_rays), ("mip_sample", mip_sample), ("mip_resample", mip_resample), ("mip_encode", mip_encode),
                     ("mip_composite_fwd", mip_composite_fwd), ("mip_composite_loss_bwd", mip_composite_loss_bwd)):
        monkeypatch.setattr(real_ops, name, fn)
    return fake
