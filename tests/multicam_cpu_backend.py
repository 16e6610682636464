"""The multiscale Mip-NeRF operators (ops.mip_rays_multi, ops.mip_encode at 16 degrees) restated from the reference's numpy / Jittor code
(contrib/mipnerf dataset/nerf.py, utils/miputils.py).  Installed over jnerf_b200.ops on top of tests/mip_cpu_backend.py so that Blenders /
Multicam / MipRunner run without a GPU, and the references the GPU tests compare the kernels against."""
import numpy as np
import torch

import mip_cpu_backend


def nerf_py_rays(images, cams, focal, white_bkgd):
    """dataset/nerf.py:152-204 (focal = 0: Multicam, pix2cam) or :265-314 (Blenders, focal) for every pixel of every image, in numpy as the
    reference writes it, images concatenated -> (rays (P, 12), target (P, 3), lossmult (P,)) float32.  images: [(H, W, 4) uint8 or fp32],
    cams: (n, 24) table rows (plugin/mip.py: cam_row)."""
    rays, targets, mults = [], [], []
    for im, c in zip(images, np.asarray(cams, np.float32)):
        h, w = im.shape[:2]
        p2c, c2w = c[0:9].reshape(3, 3), c[9:21].reshape(3, 4)
        if focal:
            x, y = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32), indexing="xy")
            f = np.float64(focal)              # .5 * w / np.tan(.5 * camera_angle_x): an fp64 scalar, so numpy computes these in fp64
            cam = np.stack([(x - w * 0.5 + 0.5) / f, -(y - h * 0.5 + 0.5) / f, -np.ones_like(x)], -1)
        else:
            x, y = np.meshgrid(np.arange(w, dtype=np.float32) + .5, np.arange(h, dtype=np.float32) + .5, indexing="xy")
            cam = np.stack([x, y, np.ones_like(x)], -1) @ p2c[:3, :3].T
        d = cam @ c2w[:3, :3].T
        o = np.broadcast_to(c2w[:3, -1], d.shape)
        v = d / np.linalg.norm(d, axis=-1, keepdims=True)
        dx = np.sqrt(np.sum((d[:-1, :, :] - d[1:, :, :]) ** 2, -1))
        dx = np.concatenate([dx, dx[-2:-1, :]], 0)
        radii = dx[..., None] * 2 / np.sqrt(12)
        ones = np.ones_like(radii)
        rays.append(np.concatenate([o, d, v, radii, ones * c[22], ones * c[23]], -1).astype(np.float32).reshape(-1, 12))
        img = im.astype(np.float32) / 255. if im.dtype == np.uint8 else im
        rgb = img[..., :3] * img[..., -1:] + (1. - img[..., -1:]) if white_bkgd else img[..., :3]
        targets.append(rgb.reshape(-1, 3).astype(np.float32))
        mults.append(np.full(h * w, c[21], np.float32))
    return np.concatenate(rays), np.concatenate(targets), np.concatenate(mults)


def install(monkeypatch):
    fake = mip_cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops
    cache = {}

    def mip_rays_multi(pix, table, focal, white_bkgd):
        fake._log("mip_rays_multi")
        key = (id(table["images"]), float(focal), bool(white_bkgd))
        if key not in cache:
            off, wh = table["offsets"].tolist(), table["wh"].tolist()
            flat = table["images"].numpy()
            images = [flat[off[i]:off[i + 1]].reshape(wh[i][1], wh[i][0], 4) for i in range(len(wh))]
            cache[key] = [torch.from_numpy(a) for a in nerf_py_rays(images, table["cams"].numpy(), focal, white_bkgd)]
        idx = pix.long()
        return tuple(a[idx] for a in cache[key])

    def mip_encode(rays, t, ray_shape="cone", integrate=True, min_deg=0, degs=8):
        fake._log("mip_encode")
        enc, view = mip_cpu_backend.encode(rays, t, ray_shape, integrate, min_deg, min_deg + degs)
        return enc.reshape(-1, 6 * degs), view

    monkeypatch.setattr(real_ops, "mip_rays_multi", mip_rays_multi)
    monkeypatch.setattr(real_ops, "mip_encode", mip_encode)
    return fake
