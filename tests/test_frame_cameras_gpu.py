"""Captures whose frames carry their own cameras on the H100: ngp_raygen_cams / ngp_prepare_batch_cams against the fp64 camera model on
frames of three sizes, bit for bit against the existing entry points on frames of one size, the occupancy grid's per-frame frustum test,
and training end to end through NerfDataset(per_frame_cameras=True)."""
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
# landscape, portrait, and a zoomed landscape frame with an off-centre principal point: (W, H, fx, fy, cx, cy)
CAMS = [(320, 180, 260.0, 262.0, 160.0, 90.0), (180, 320, 250.0, 249.0, 92.5, 158.0), (320, 180, 540.0, 538.0, 96.0, 117.0)]
LENSES = [FOX_LENS, (0.0, 0.0, 0.0, 0.0), (-0.08, 0.01, 0.001, -0.002)]


def random_xforms(n, seed):
    """(n, 12) column-major camera-to-world tables of random rotations, as NerfDataset stores them."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        m = np.concatenate([q * np.sign(np.linalg.det(q)), rng.uniform(0, 1, (3, 1))], 1).astype(np.float32)
        out.append(np.ascontiguousarray(m.T).reshape(12))
    return torch.from_numpy(np.stack(out)).cuda()


def capture(cams, lenses=None, seed=0):
    """The device tables of a ragged capture: (offsets, wh, xforms, focal, principal, distortion or None)."""
    wh = np.array([c[:2] for c in cams], np.int64)
    offsets = np.concatenate([[0], np.cumsum(wh[:, 0] * wh[:, 1])])
    focal = torch.tensor([c[2:4] for c in cams], dtype=torch.float32, device="cuda")
    principal = torch.tensor([[c[4] / c[0], c[5] / c[1]] for c in cams], dtype=torch.float32, device="cuda")
    dist = None if lenses is None else torch.tensor(lenses, dtype=torch.float32, device="cuda")
    return (torch.from_numpy(offsets.astype(np.int32)).cuda(), torch.from_numpy(wh.astype(np.int32)).cuda(), random_xforms(len(cams), seed),
            focal, principal, dist)


def pixel_error(rays_d, pix, offsets, wh, xforms, focal, principal, lenses):
    """|pixel the ray is seen at - the centre of the pixel it was made for| in pixels: the kernel direction in its image's camera axes
    (the fp32 table solved in fp64), projected and sent through the fp64 lens model; the image and pixel from the prefix sums."""
    pix = pix.long().cpu().numpy()
    off_all, wh = offsets.long().cpu().numpy(), wh.long().cpu().numpy()
    ids = np.searchsorted(off_all, pix, side="right") - 1
    m = xforms.double().cpu().numpy().reshape(-1, 4, 3)
    d = rays_d.double().cpu().numpy()
    err = np.zeros(len(pix))
    for i in np.unique(ids):
        s = ids == i
        W, H = wh[i]
        off = pix[s] - off_all[i]
        c = np.linalg.solve(m[i, :3].T, d[s].T).T
        x, y = c[:, 0] / c[:, 2], c[:, 1] / c[:, 2]
        if lenses is not None:
            x, y = D.lens_distort(x, y, lenses[i])
        f, p = focal[i].double().cpu().numpy(), principal[i].double().cpu().numpy()
        u, v = x * f[0] + p[0] * W, y * f[1] + p[1] * H
        err[s] = np.hypot(u - (off % W + 0.5), v - (off // W + 0.5))
    return err


@pytest.mark.parametrize("lens", [False, True], ids=["pinhole", "lens"])
def test_cams_rays_land_on_their_pixels_and_targets_are_the_ragged_pixels(lens):
    """Every pixel of six frames of three sizes (landscape, portrait, zoomed with an off-centre principal point): each ray of
    ngp_raygen_cams lands within 1e-3 px of its pixel's centre through the fp64 model (the bound of test_lens_gpu.py: a few fp32 ulps of
    the pixel coordinate and of the direction).  ngp_prepare_batch_cams gives the same rays bit for bit, and its targets are the ragged
    table's pixels blended over bg, for uint8 and f32 tables, to within the rounding of the blend's one multiply-add."""
    cams = CAMS * 2
    lenses = (LENSES * 2) if lens else None
    offsets, wh, xf, focal, principal, dist = capture(cams, lenses)
    total = int(offsets[-1])
    pix = torch.arange(total, dtype=torch.int32, device="cuda")
    ids, o, d = ops.raygen_cams(pix, offsets, wh, xf, focal, principal, distortion=dist)
    err = pixel_error(d, pix, offsets, wh, xf, focal, principal, lenses)
    assert err.max() < 1e-3, (err.max(), np.median(err))
    want_ids = torch.repeat_interleave(torch.arange(len(cams), device="cuda", dtype=torch.int32), (wh[:, 0] * wh[:, 1]).long())
    assert torch.equal(ids, want_ids) and torch.equal(o, xf.reshape(-1, 4, 3)[ids.long(), 3])
    g = torch.Generator(device="cuda").manual_seed(3)
    perm = torch.randperm(total, device="cuda", generator=g).int()
    bg = torch.rand((total, 3), device="cuda", generator=g)
    img8 = torch.randint(0, 256, (total, 4), device="cuda", generator=g, dtype=torch.uint8)
    img32 = torch.rand((total, 4), device="cuda", generator=g)
    for img in (img8, img32):
        b_ids, b_o, b_d, target = ops.prepare_batch_cams(perm, offsets, wh, xf, focal, principal, img, bg, distortion=dist)
        k = perm.long()
        assert torch.equal(b_ids, ids[k]) and torch.equal(b_o, o[k]) and torch.equal(b_d, d[k])
        c = img[k].float() / 255.0 if img.dtype == torch.uint8 else img[k]
        want = c[:, :3] * c[:, 3:] + bg * (1 - c[:, 3:])
        assert (target - want).abs().max() <= 2 ** -22, (target - want).abs().max()


@pytest.mark.parametrize("lens", [False, True], ids=["pinhole", "lens"])
def test_cams_on_frames_of_one_size_are_the_existing_entry_points_bit_for_bit(lens):
    """Five 54x96 frames with their own focal lengths, principal points and lenses: raygen_cams / prepare_batch_cams give the rays and
    targets of raygen / prepare_batch (the _lens ones with a lens) bit for bit, on 2^18 random pixels, for uint8 and f32 images."""
    n_img, W, H, n = 5, 54, 96, 1 << 18
    g = torch.Generator(device="cuda").manual_seed(0)
    xf = random_xforms(n_img, 0)
    focal = torch.tensor([[75.0, 74.5]] * n_img, device="cuda") + torch.rand((n_img, 2), device="cuda", generator=g)
    principal = 0.5 + 0.02 * torch.rand((n_img, 2), device="cuda", generator=g)
    dist = torch.tensor([FOX_LENS, (0.25, 0, 0, 0), (0.1, -0.05, 0.002, -0.003), FOX_LENS, (-0.08, 0.01, 0.0, 0.001)], device="cuda") if lens else None
    pix = torch.randint(0, n_img * H * W, (n,), device="cuda", generator=g, dtype=torch.int32)
    bg = torch.rand((n, 3), device="cuda", generator=g)
    offsets = (torch.arange(n_img + 1, device="cuda") * (H * W)).int()
    wh = torch.tensor([[W, H]] * n_img, dtype=torch.int32, device="cuda")
    kw = {} if dist is None else dict(distortion=dist)
    a = ops.raygen(pix, W, H, xf, focal, principal, **kw)
    b = ops.raygen_cams(pix, offsets, wh, xf, focal, principal, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for img in (torch.randint(0, 256, (n_img, H * W, 4), device="cuda", generator=g, dtype=torch.uint8),
                torch.rand((n_img, H * W, 4), device="cuda", generator=g)):
        a = ops.prepare_batch(pix, W, H, xf, focal, principal, img, bg, **kw)
        b = ops.prepare_batch_cams(pix, offsets, wh, xf, focal, principal, img, bg, **kw)
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def morton_invert(x):
    x = x & 0x49249249
    x = (x | (x >> 2)) & 0xC30C30C3
    x = (x | (x >> 4)) & 0x0F00F00F
    x = (x | (x >> 8)) & 0xFF0000FF
    return (x | (x >> 16)) & 0x0000FFFF


def visible_cells(xforms, cams, lenses, cascades=5, n=128 ** 3):
    """The fp64 restatement of visibility: a cell whose centre some frame sees through one of its pixels -- in front of the camera, and
    projected through the frame's forward lens model inside its W x H image, out to where the lens folds over."""
    idx = torch.arange(n, device="cuda", dtype=torch.int64)
    xyz = torch.stack([morton_invert(idx >> k) for k in range(3)], -1).double()
    m = xforms.double().reshape(-1, 4, 3)
    visible = torch.zeros(cascades * n, dtype=torch.bool, device="cuda")
    for level in range(cascades):
        p = ((xyz + 0.5) / 128 - 0.5) * 2.0 ** level + 0.5
        vis = torch.zeros(n, dtype=torch.bool, device="cuda")
        for j, (W, H, fx, fy, cx, cy) in enumerate(cams):
            k1, k2, p1, p2 = lenses[j] if lenses else (0.0, 0.0, 0.0, 0.0)
            roots = [t.real for t in np.roots([5 * k2, 3 * k1, 1.0]) if abs(t.imag) < 1e-12 and t.real > 0] if k2 else ([-1 / (3 * k1)] if k1 < 0 else [])
            r2_max = 0.9 * min(roots) if roots else math.inf
            c = (p - m[j, 3]) @ m[j, :3].T
            z = c[:, 2]
            x, y = c[:, 0] / z, c[:, 1] / z
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            xd, yd = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
            u, v = xd * fx + cx, yd * fy + cy
            vis |= (z > 0) & (r2 < r2_max) & (u >= 0) & (u <= W) & (v >= 0) & (v <= H)
        visible[level * n:(level + 1) * n] = vis
    return visible


@pytest.mark.parametrize("lens", [False, True], ids=["pinhole", "lens"])
def test_every_cell_a_pixel_of_some_frame_sees_is_trainable(lens):
    """ngp_grid_mark_untrained_cams with the dataset's frame_extents marks every cell some frame sees (visible_cells) trainable.  For
    the zoomed frame alone, the symmetric test of ngp_grid_mark_untrained misses cells its off-centre principal point shows."""
    cams = [tuple(c) for c in CAMS] * 3
    lenses = LENSES * 3 if lens else None
    ds = D.SyntheticNerfDataset(n_images=9, batch_size=4096, seed=2, style="fox",
                                cameras=[c + (k,) for c, k in zip(cams, lenses)] if lens else cams, undistort=lens)
    assert ds.frame_cameras
    g = torch.zeros(5 * 128 ** 3, device="cuda")
    ops.grid_mark_untrained_cams(g, ds.frame_extents, ds.transforms_gpu)
    visible = visible_cells(ds.transforms_gpu, cams, lenses)
    assert int(visible.sum()) > 10000
    assert bool((g[visible] == 0).all()), int((g[visible] != 0).sum())
    z = [2]
    xf = ds.transforms_gpu[z].contiguous()
    zoomed = [cams[2]]
    vis = visible_cells(xf, zoomed, [lenses[2]] if lens else None)
    old = torch.zeros_like(g)
    ops.grid_mark_untrained(old, ds.focal_lengths[z].contiguous(), xf, zoomed[0][:2])
    new = torch.zeros_like(g)
    ops.grid_mark_untrained_cams(new, ds.frame_extents[z].contiguous(), xf)
    assert bool((new[vis] == 0).all()) and int((old[vis] != 0).sum()) > 0


def fox_small(tmp_path):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_fox_small import materialise
    return materialise(str(tmp_path / "fox"))


def nerf_runner(root, per_frame, undistort=False, seed=1, style="fox", **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    make = fox_cfg if style == "fox" else lego_cfg
    c = make(fp16=True, synthetic=False, seed=seed, **over)
    for split in list(c["dataset"]):
        if c["dataset"][split] is None:
            continue
        c["dataset"][split].update(root_dir=root, **({"per_frame_cameras": True} if per_frame else {}), **({"undistort": True} if undistort else {}))
    if style != "fox":
        c["dataset"]["val"] = dict(c["dataset"]["test"])
    update_cfg(**c)
    return Runner()


def state(r):
    r._table_ready()
    m, s = r.model, r.sampler
    return [t.detach().clone() for t in (m.pos_encoder.m_grid, m.density_mlp.con_weights, m.rgb_mlp.con_weights, s.density_grid,
                                         s.density_grid_bitfield)]


def test_per_frame_keyword_on_one_camera_trains_bit_identically(tmp_path, monkeypatch):
    """fox_small has no per-frame keys: per_frame_cameras=True (with undistort, so the lens path runs too) takes the existing entry
    points and 50 seeded steps end with the parameters and occupancy grid of the keyword off, bit for bit."""
    root = fox_small(tmp_path)
    names = []
    call = lib.call
    monkeypatch.setattr(lib, "call", lambda name, *a: names.append(name) or call(name, *a))
    out = []
    for per_frame in (False, True):
        r = nerf_runner(root, per_frame, undistort=True)
        assert not r.dataset["train"].frame_cameras
        for _ in range(50):
            r.train_step()
        out.append(state(r))
        del r
    assert not any(n.endswith("_cams") for n in names) and "ngp_prepare_batch_lens" in names
    assert all(torch.equal(a, b) for a, b in zip(*out))


def halve_every_other_frame(root):
    """fox_small with every other training frame (and the test frames that share its file) box-downscaled by 2, and every frame carrying
    its own w, h, fl_x, fl_y, cx, cy.  Frames whose file is missing are dropped, as NerfDataset drops them."""
    from PIL import Image
    jds = {split: json.load(open(os.path.join(root, f"transforms_{split}.json"))) for split in ("train", "test")}
    for jd in jds.values():
        jd["frames"] = [fr for fr in jd["frames"] if os.path.exists(os.path.join(root, fr["file_path"]))]
    halved = {fr["file_path"] for i, fr in enumerate(jds["train"]["frames"]) if i % 2}
    for name in halved:
        f = os.path.join(root, name)
        im = Image.open(f)
        im.resize((im.width // 2, im.height // 2), Image.BOX).save(f, quality=95)
    for split, jd in jds.items():
        for fr in jd["frames"]:
            s = 2 if fr["file_path"] in halved else 1
            im = Image.open(os.path.join(root, fr["file_path"]))
            fr.update(w=im.width, h=im.height, fl_x=jd["fl_x"] / s, fl_y=jd["fl_y"] / s, cx=jd["cx"] / s, cy=jd["cy"] / s)
        json.dump(jd, open(os.path.join(root, f"transforms_{split}.json"), "w"))
    return root


def test_fox_small_with_every_other_frame_halved(tmp_path):
    """The reduced fox capture with every other frame at half size: every ray of every frame lands on its pixel through the frame's own
    camera and the capture's lens, and 300 training steps raise the held-out PSNR by more than 2 dB."""
    root = halve_every_other_frame(fox_small(tmp_path))
    for split in ("train", "test"):
        ds = D.NerfDataset(root, 4096, mode=split, per_frame_cameras=True, undistort=True)
        assert ds.frame_cameras and {tuple(r) for r in ds.resolutions.tolist()} == {(180, 320), (90, 160)}
        pix = torch.arange(ds.total_pixels, dtype=torch.int32, device="cuda")
        _, _, d = ds.rays_for(pix)
        err = pixel_error(d, pix, ds.pixel_offsets, ds.resolutions, ds.transforms_gpu, ds.focal_lengths, ds.principal,
                          ds.distortion.double().cpu().numpy())
        assert err.max() < 1e-3, (split, err.max())
    r = nerf_runner(root, True, undistort=True)
    r.dataset["val"] = D.NerfDataset(root, 4096, mode="test", per_frame_cameras=True, undistort=True, preload_shuffle=False)
    assert r.dataset["val"].frame_cameras
    before = r.psnr("val")
    for _ in range(300):
        r.train_step()
    after = r.psnr("val")
    print("fox_small halved frames held-out PSNR:", before, after)
    assert after > before + 2.0, (before, after)


# The mixed stand-in (lego scene: frames cycling through a 200x200 camera, a 240x160 one and a 160x240 one zoomed 1.5x with an
# off-centre principal point) against the same scene with one 200x200 camera, both trained E2E_STEPS seeded steps.  Measured once on an
# H100 SXM (80 GB HBM3, 700 W power limit, SM clock limit 1980 MHz): 31.25 dB mixed, 31.72 dB one camera, a gap of 0.47 dB; the margin
# is about three times that.
E2E_STEPS = 1500
E2E_MARGIN_DB = 1.5
MIXED = [(200, 200, 280.0, 280.0, 100.0, 100.0), (240, 160, 300.0, 300.0, 120.0, 80.0), (160, 240, 420.0, 420.0, 56.0, 150.0)]


def test_mixed_stand_in_end_to_end(tmp_path):
    """Train the mixed stand-in through write_synthetic_frames and NerfDataset(per_frame_cameras=True); test() writes every held-out view
    at its own size and its mean PSNR is the mean of the per-view PSNRs; the held-out PSNR is within E2E_MARGIN_DB of the same scene
    taken with one camera."""
    from PIL import Image
    from jnerf_b200.plugin import losses as L
    root = str(tmp_path / "mixed")
    src = D.write_synthetic_frames(root, MIXED, n_images=60)
    res = {}
    r = nerf_runner(root, True, style="lego", log_dir=str(tmp_path / "logs"), exp_name="mixed")
    assert r.dataset["train"].frame_cameras
    for _ in range(E2E_STEPS):
        r.train_step()
    seen = {}
    render_test = r.render_test
    r.render_test = lambda *a, **k: seen.setdefault("mse", render_test(*a, **k))
    psnr = r.test()
    test_ds = r.dataset["test"]
    for i in range(test_ds.n_images):
        w, h = test_ds.image_resolution(i)
        for kind in ("r", "gt"):
            assert Image.open(str(tmp_path / "logs" / "mixed" / "test" / f"mixed_{kind}_{i}.png")).size == (w, h)
    per_view = [float(L.mse2psnr(torch.tensor(v)).item()) for v in seen["mse"]]
    assert abs(psnr - sum(per_view) / len(per_view)) < 1e-9 and {test_ds.image_resolution(i) for i in range(test_ds.n_images)} == \
        {c[:2] for c in MIXED[:test_ds.n_images]}
    res["mixed"] = psnr
    del r
    torch.cuda.empty_cache()
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    c = lego_cfg(fp16=True, synthetic=True, seed=1, log_dir=str(tmp_path / "logs"), exp_name="one")
    for split in ("train", "val", "test"):
        c["dataset"][split].update(n_images=60, cameras=[MIXED[0]])
    update_cfg(**c)
    r = Runner()
    for _ in range(E2E_STEPS):
        r.train_step()
    res["one"] = r.test()
    print("per-frame cameras e2e held-out PSNR:", json.dumps(res))
    assert src["test"].n_images == 6
    assert res["one"] - res["mixed"] < E2E_MARGIN_DB, res
