"""Lens distortion on the H100: ngp_raygen_lens / ngp_prepare_batch_lens against an fp64 restatement of the lens model, their bit-level
relations to each other and to the pinhole entry points, the occupancy grid's visibility through a lens, and training end to end on a
stand-in whose images were taken through a strong lens."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

from jnerf_b200 import lib, ops
from jnerf_b200.plugin import dataset as D

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FOX_LENS = (0.0578421, -0.0805099, -0.000980296, 0.00015575)          # data/fox/transforms_train.json
FOX = dict(W=1080, H=1920, fl=(1375.52, 1374.49), c=(554.558, 965.268))
STRONG = (0.25, 0.0, 0.0, 0.0)


def random_xforms(n, seed):
    """(n, 12) column-major camera-to-world tables of random rotations, as NerfDataset stores them."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        m = np.concatenate([q * np.sign(np.linalg.det(q)), rng.uniform(0, 1, (3, 1))], 1).astype(np.float32)
        out.append(np.ascontiguousarray(m.T).reshape(12))
    return torch.from_numpy(np.stack(out)).cuda()


def pixel_error(rays_d, pix, W, H, xforms, focal, principal, lens):
    """|pixel the ray is seen at - the pixel's centre| in pixels: the kernel direction in the camera's axes (the fp32 table solved in
    fp64), projected and sent through the fp64 forward model."""
    pix = pix.long().cpu().numpy()
    ids, off = pix // (H * W), pix % (H * W)
    m = xforms.double().cpu().numpy().reshape(-1, 4, 3)                            # rows: camera x, y, z axes, origin
    d = rays_d.double().cpu().numpy()
    err = np.zeros(len(pix))
    for i in np.unique(ids):
        s = ids == i
        c = np.linalg.solve(m[i, :3].T, d[s].T).T                                   # d = c0 x_axis + c1 y_axis + c2 z_axis
        xd, yd = D.lens_distort(c[:, 0] / c[:, 2], c[:, 1] / c[:, 2], lens[i])
        f, p = focal[i].double().cpu().numpy(), principal[i].double().cpu().numpy()
        u, v = xd * f[0] + p[0] * W, yd * f[1] + p[1] * H
        err[s] = np.hypot(u - (off[s] % W + 0.5), v - (off[s] // W + 0.5))
    return err


@pytest.mark.parametrize("lens", [FOX_LENS, STRONG], ids=["fox", "k1=0.25"])
def test_lens_rays_land_on_their_pixels_full_frame(lens):
    """Every pixel of two 1080x1920 frames with the fox capture's intrinsics: each ray of ngp_raygen_lens, mapped back through the fp64
    forward model, lands within 1e-3 px of its pixel centre.  The bound is derived: the fp32 pixel coordinate (x - cx) W / fx and the
    fp32 direction each carry a few ulps of a coordinate of order 1, 6e-8 x 1375 px = 8e-5 px apiece, about 1.4e-4 px together; 1e-3 px
    leaves room for the Newton solve's last step, and a lens ignored (the pinhole ray) misses by up to 10.8 px."""
    W, H, n = FOX["W"], FOX["H"], 2
    D.check_lens(lens, W, H, FOX["fl"], FOX["c"])
    xf = random_xforms(n, 3)
    focal = torch.tensor([FOX["fl"]] * n, dtype=torch.float32, device="cuda")
    principal = torch.tensor([[FOX["c"][0] / W, FOX["c"][1] / H]] * n, dtype=torch.float32, device="cuda")
    dist = torch.tensor([lens] * n, dtype=torch.float32, device="cuda")
    pix = torch.arange(n * H * W, dtype=torch.int32, device="cuda")
    _, _, d = ops.raygen(pix, W, H, xf, focal, principal, distortion=dist)
    err = pixel_error(d, pix, W, H, xf, focal, principal, [lens] * n)
    assert err.max() < 1e-3, (err.max(), np.median(err))
    _, _, d0 = ops.raygen(pix, W, H, xf, focal, principal)
    assert pixel_error(d0, pix, W, H, xf, focal, principal, [lens] * n).max() > 1.0      # the pinhole ray is far off


def test_fox_small_capture_rays_land_on_their_pixels(tmp_path):
    """The reduced fox capture through NerfDataset(undistort=True): every pixel of every test and training image."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_fox_small import materialise
    root = materialise(str(tmp_path / "fox"))
    for split in ("train", "test"):
        ds = D.NerfDataset(root, 4096, mode=split, undistort=True)
        lens = ds.distortion.cpu().numpy().astype(np.float64)
        pix = torch.arange(ds.n_images * ds.H * ds.W, dtype=torch.int32, device="cuda")
        _, _, d = ds.rays_for(pix)
        err = pixel_error(d, pix, ds.W, ds.H, ds.transforms_gpu, ds.focal_lengths, ds.principal, lens)
        assert err.max() < 1e-3, (split, err.max())
        o, d1 = ds.generate_rays_total_test(1)
        assert torch.equal(d1, d[ds.H * ds.W:2 * ds.H * ds.W])


def batch_inputs(n_img=5, H=96, W=54, n=1 << 18, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xf = random_xforms(n_img, seed)
    focal = torch.tensor([[75.0, 74.5]] * n_img, device="cuda") + torch.rand((n_img, 2), device="cuda", generator=g)
    principal = 0.5 + 0.02 * torch.rand((n_img, 2), device="cuda", generator=g)
    dist = torch.tensor([FOX_LENS, STRONG, (0.1, -0.05, 0.002, -0.003), FOX_LENS, (-0.08, 0.01, 0.0, 0.001)][:n_img], device="cuda")
    pix = torch.randint(0, n_img * H * W, (n,), device="cuda", generator=g, dtype=torch.int32)
    img8 = torch.randint(0, 256, (n_img, H * W, 4), device="cuda", generator=g, dtype=torch.uint8)
    img32 = torch.rand((n_img, H * W, 4), device="cuda", generator=g)
    bg = torch.rand((n, 3), device="cuda", generator=g)
    return pix, W, H, xf, focal, principal, dist, img8, img32, bg


def test_prepare_batch_lens_is_raygen_lens_plus_the_pinhole_targets():
    """ngp_prepare_batch_lens: rays bit for bit those of ngp_raygen_lens, targets bit for bit those of ngp_prepare_batch, and two runs
    identical -- for uint8 and f32 images, with a different lens on every image."""
    pix, W, H, xf, focal, principal, dist, img8, img32, bg = batch_inputs()
    ids, o, d = ops.raygen(pix, W, H, xf, focal, principal, distortion=dist)
    for img in (img8, img32):
        a = ops.prepare_batch(pix, W, H, xf, focal, principal, img, bg, distortion=dist)
        b = ops.prepare_batch(pix, W, H, xf, focal, principal, img, bg, distortion=dist)
        pin = ops.prepare_batch(pix, W, H, xf, focal, principal, img, bg)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        assert torch.equal(a[0], ids) and torch.equal(a[1], o) and torch.equal(a[2], d)
        assert torch.equal(a[3], pin[3]) and torch.equal(a[0], pin[0]) and torch.equal(a[1], pin[1]) and not torch.equal(a[2], pin[2])
    err = pixel_error(d[:20000], pix[:20000], W, H, xf, focal, principal, dist.double().cpu().numpy())
    assert err.max() < 1e-3


def test_a_zero_lens_takes_the_pinhole_entry_points_bit_for_bit(monkeypatch):
    pix, W, H, xf, focal, principal, dist, img8, _, bg = batch_inputs(seed=1)
    names = []
    call = lib.call
    monkeypatch.setattr(lib, "call", lambda name, *a: names.append(name) or call(name, *a))
    zero = torch.zeros_like(dist)
    r0, r1 = ops.raygen(pix, W, H, xf, focal, principal), ops.raygen(pix, W, H, xf, focal, principal, distortion=zero)
    p0, p1 = (ops.prepare_batch(pix, W, H, xf, focal, principal, img8, bg),
              ops.prepare_batch(pix, W, H, xf, focal, principal, img8, bg, distortion=zero))
    assert names == ["ngp_raygen", "ngp_raygen", "ngp_prepare_batch", "ngp_prepare_batch"]
    assert all(torch.equal(x, y) for x, y in zip(r0 + p0, r1 + p1))


def fox_runner(undistort, distortion=None, n_images=6, H=160, W=90, seed=1, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**fox_cfg(fp16=True, synthetic=True, undistort=undistort, seed=seed, **over))
    cfg = get_cfg()
    for split in ("train", "test"):
        d = cfg.dataset[split]
        d.n_images, d.H, d.W = n_images, H, W
        if distortion is not None:
            d.distortion = list(distortion)
    cfg.dataset.val = dict(cfg.dataset.test)                           # the held-out views, for Runner.psnr("val")
    return Runner()


def test_undistort_on_a_zero_lens_capture_trains_bit_identically():
    """50 seeded steps of the fox configuration on a pinhole stand-in: undistort=True (a lens of zeros) and undistort=False end with the
    same parameters and occupancy grid, bit for bit."""
    out = []
    for undistort in (False, True):
        r = fox_runner(undistort)
        assert (r.dataset["train"].distortion is not None) == undistort
        for _ in range(50):
            r.train_step()
        r._table_ready()
        m, s = r.model, r.sampler
        out.append([t.detach().clone() for t in (m.pos_encoder.m_grid, m.density_mlp.con_weights, m.rgb_mlp.con_weights, s.density_grid,
                                                 s.density_grid_bitfield)])
    assert all(torch.equal(a, b) for a, b in zip(*out))


def morton_invert(x):
    x = x & 0x49249249
    x = (x | (x >> 2)) & 0xC30C30C3
    x = (x | (x >> 4)) & 0x0F00F00F
    x = (x | (x >> 8)) & 0xFF0000FF
    return (x | (x >> 16)) & 0x0000FFFF


@pytest.mark.parametrize("lens", [FOX_LENS, (-0.12, 0.01, 0.001, -0.002)], ids=["fox", "barrel"])
def test_every_cell_a_pixel_sees_through_the_lens_is_trainable(lens):
    """ngp_grid_mark_untrained with the dataset's focal_eff, against the fp64 restatement of visibility: a cell whose centre a camera
    sees through one of its pixels (in front of it, and projected through the forward lens model inside the image) must be marked
    trainable (0).  With a barrel lens the images see beyond the pinhole frustum of their focal lengths: that frustum misses cells."""
    ds = D.SyntheticNerfDataset(style="fox", H=192, W=108, n_images=10, distortion=lens, undistort=True, seed=2)
    cascades = 5
    n = 128 ** 3
    grids = {}
    for name, focal in (("eff", ds.focal_eff), ("pinhole", ds.focal_lengths)):
        g = torch.zeros(cascades * n, device="cuda")
        ops.grid_mark_untrained(g, focal, ds.transforms_gpu, ds.resolution)
        grids[name] = g
    # the forward model is one to one out to the first zero of d/dr r (1 + k1 r^2 + k2 r^4) (check_lens vouches for the image inside it);
    # beyond it a direction far outside the image can map back into it
    k1, k2, p1, p2 = lens
    roots = [t.real for t in np.roots([5 * k2, 3 * k1, 1.0]) if abs(t.imag) < 1e-12 and t.real > 0] if k2 else ([-1 / (3 * k1)] if k1 < 0 else [])
    r2_max = 0.9 * min(roots) if roots else math.inf
    idx = torch.arange(n, device="cuda", dtype=torch.int64)
    xyz = torch.stack([morton_invert(idx >> k) for k in range(3)], -1).double()
    m = ds.transforms_gpu.double().reshape(-1, 4, 3)
    fx, fy = ds._focal
    visible = torch.zeros(cascades * n, dtype=torch.bool, device="cuda")
    for level in range(cascades):
        p = ((xyz + 0.5) / 128 - 0.5) * 2.0 ** level + 0.5
        vis = torch.zeros(n, dtype=torch.bool, device="cuda")
        for j in range(ds.n_images):
            c = (p - m[j, 3]) @ m[j, :3].T                                           # camera x, y, z of every cell centre
            z = c[:, 2]
            front = z > 0
            x, y = c[:, 0] / z, c[:, 1] / z
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            xd, yd = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
            u, v = xd * fx + ds._cx, yd * fy + ds._cy
            ok = front & (r2 < r2_max) & (u >= 0) & (u <= ds.W) & (v >= 0) & (v <= ds.H)
            vis |= ok
        visible[level * n:(level + 1) * n] = vis
    assert int(visible.sum()) > 10000
    assert bool((grids["eff"][visible] == 0).all()), int((grids["eff"][visible] != 0).sum())
    if lens[0] < 0:
        assert int((grids["pinhole"][visible] != 0).sum()) > 0


# Held-out PSNR measured once on an H100 SXM (80 GB HBM3, 700 W power limit, SM clock 1980 MHz): undistort=True 28.08 dB, undistort=False
# 23.05 dB, no lens 29.97 dB -- a gain of 5.03 dB and a gap of 1.89 dB.  The thresholds leave about 2 dB and 1.6 dB of headroom.
PSNR_GAIN_MIN = 3.0
PSNR_GAP_MAX = 3.5


def test_training_through_a_strong_lens_end_to_end():
    """A reduced fox stand-in whose images were taken through k1 = 0.25, trained 1500 seeded steps with undistort=True and with
    undistort=False, and the same scene without a lens; held-out views rendered through the lens (render_img).  Measured once on the
    H100: 28.08 dB with undistort=True, 23.05 dB with undistort=False (its renders are pinhole images scored against photos taken
    through the lens), 29.97 dB without a lens.  Undistorting must gain more than PSNR_GAIN_MIN and come within PSNR_GAP_MAX of the
    lens-free scene."""
    steps, kw = 1500, dict(n_images=30, H=288, W=162, seed=1)
    res = {}
    for name, undistort, lens in (("on", True, STRONG), ("off", False, STRONG), ("none", False, None)):
        r = fox_runner(undistort, lens, **kw)
        for _ in range(steps):
            r.train_step()
        res[name] = r.psnr("val")
        del r
        torch.cuda.empty_cache()
    print("lens e2e held-out PSNR:", json.dumps(res))
    assert res["on"] - res["off"] > PSNR_GAIN_MIN, res
    assert res["none"] - res["on"] < PSNR_GAP_MAX, res
