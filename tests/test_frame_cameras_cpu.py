"""Instant-NGP captures whose frames carry their own cameras (`per_frame_cameras=True`), without a GPU: how a frame's keys override the
json's top level, the refusals per frame, the ragged pixel table and its shuffle, the frustum extents of the occupancy grid, and which
entry points every batch, render and grid update calls -- on every data-parallel rank -- while a capture whose frames share one camera
loads and trains exactly as with the keyword off.  The `_cams` kernels themselves are checked on the GPU (test_frame_cameras_gpu.py)."""
import json
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from jnerf_b200 import ops
from jnerf_b200.plugin import dataset as D

HERE = os.path.dirname(os.path.abspath(__file__))


def frame_rays(pix, offsets, wh, xforms, focal, principal, distortion=None):
    """The rays of ngp_raygen_cams restated in fp64: pixel id -> image by a search over the prefix sums, -> (x, y) in that image,
    -> the normalised coordinate, undistorted by a fixed-point iteration, -> the direction through the camera's axes."""
    pix = pix.long().numpy()
    off_all, wh = offsets.long().numpy(), wh.long().numpy()
    ids = np.searchsorted(off_all, pix, side="right") - 1
    W, H = wh[ids, 0], wh[ids, 1]
    off = pix - off_all[ids]
    m = xforms.double().numpy().reshape(-1, 4, 3)[ids]                              # rows: camera x, y, z axes, origin
    xd = ((off % W) + 0.5 - principal[ids, 0].double().numpy() * W) / focal[ids, 0].double().numpy()
    yd = ((off // W) + 0.5 - principal[ids, 1].double().numpy() * H) / focal[ids, 1].double().numpy()
    x, y = xd.copy(), yd.copy()
    if distortion is not None:
        k1, k2, p1, p2 = distortion.double().numpy()[ids].T
        for _ in range(200):
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            x, y = (xd - 2 * p1 * x * y - p2 * (r2 + 2 * x * x)) / rad, (yd - p1 * (r2 + 2 * y * y) - 2 * p2 * x * y) / rad
    d = m[:, 0] * x[:, None] + m[:, 1] * y[:, None] + m[:, 2]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return torch.from_numpy(ids.astype(np.int32)), torch.from_numpy(m[:, 3].astype(np.float32)), torch.from_numpy(d.astype(np.float32))


class FrameOps:
    """CPU stand-ins of the four ray entry points of ops, computed by frame_rays; every call is recorded by name."""

    def __init__(self):
        self.calls = []

    @staticmethod
    def _contiguous(*ts):
        """The kernels take plain pointers (ops._p): every table handed to them must be contiguous."""
        assert all(t is None or t.is_contiguous() for t in ts)

    @staticmethod
    def _uniform(n, W, H):
        return torch.arange(n + 1, dtype=torch.int64) * (W * H), torch.tensor([[W, H]] * n)

    def raygen(self, pix, W, H, xforms, focal, principal, **kw):
        self._contiguous(pix, xforms, focal, principal, kw.get("distortion"))
        self.calls.append("raygen")
        return frame_rays(pix, *self._uniform(xforms.shape[0], W, H), xforms, focal, principal, ops.lens_of(kw.get("distortion")))

    def raygen_cams(self, pix, offsets, wh, xforms, focal, principal, **kw):
        self._contiguous(pix, offsets, wh, xforms, focal, principal, kw.get("distortion"))
        self.calls.append("raygen_cams")
        return frame_rays(pix, offsets, wh, xforms, focal, principal, ops.lens_of(kw.get("distortion")))

    @staticmethod
    def _target(images, pix, bg):
        rgba = images.reshape(-1, 4)[pix.long()].float() / 255.0
        return rgba[:, :3] * rgba[:, 3:] + bg * (1 - rgba[:, 3:])

    def prepare_batch(self, pix, W, H, xforms, focal, principal, images, bg, **kw):
        self._contiguous(pix, xforms, focal, principal, images, bg, kw.get("distortion"))
        self.calls.append("prepare_batch")
        img, o, d = frame_rays(pix, *self._uniform(xforms.shape[0], W, H), xforms, focal, principal, ops.lens_of(kw.get("distortion")))
        return img, o, d, self._target(images, pix, bg)

    def prepare_batch_cams(self, pix, offsets, wh, xforms, focal, principal, images, bg, **kw):
        self._contiguous(pix, offsets, wh, xforms, focal, principal, images, bg, kw.get("distortion"))
        self.calls.append("prepare_batch_cams")
        img, o, d = frame_rays(pix, offsets, wh, xforms, focal, principal, ops.lens_of(kw.get("distortion")))
        return img, o, d, self._target(images, pix, bg)

    def install(self, mp):
        for name in ("raygen", "raygen_cams", "prepare_batch", "prepare_batch_cams"):
            mp.setattr(ops, name, getattr(self, name))
        mp.setattr(D, "DEVICE", "cpu")
        return self


@pytest.fixture()
def fops(monkeypatch):
    return FrameOps().install(monkeypatch)


# three cameras: landscape, portrait, and a zoomed landscape frame with an off-centre principal point
CAMS = [dict(w=12, h=8, fl_x=11.0, fl_y=11.5, cx=6.0, cy=4.0),
        dict(w=8, h=12, fl_x=9.0, fl_y=9.0, cx=4.25, cy=5.5),
        dict(w=12, h=8, fl_x=22.0, fl_y=21.0, cx=2.5, cy=6.5)]
LENS = dict(k1=0.08, k2=-0.02, p1=0.003, p2=-0.002)


def write_capture(root, frames, top=None, n=None, seed=0):
    """A capture in the Instant-NGP layout: transforms_train.json with `top` at the top level and frame i carrying frames[i % len]'s keys;
    every image is random RGBA at the size the frame (else the top level) names."""
    from PIL import Image
    top = {} if top is None else dict(top)
    n = len(frames) if n is None else n
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    mats = D.synthetic_cameras(n, seed=seed)
    out = []
    for i in range(n):
        keys = dict(frames[i % len(frames)])
        w, h = int(keys.get("w", top.get("w"))), int(keys.get("h", top.get("h")))
        Image.fromarray(rng.integers(0, 256, (h, w, 4), dtype=np.uint8), "RGBA").save(os.path.join(root, "images", f"f{i}.png"))
        out.append(dict(file_path=f"images/f{i}", transform_matrix=mats[i].tolist(), **keys))
    with open(os.path.join(root, "transforms_train.json"), "w") as fh:
        json.dump(dict(top, frames=out), fh)
    return root


def camera_of(c, lens=None):
    return (c["w"], c["h"], c["fl_x"], c["fl_y"], c["cx"], c["cy"]) + ((lens,) if lens else ())


def test_frame_keys_override_top_level_keys(tmp_path, fops):
    """Each frame's own w, h, fl_x, fl_y, cx, cy win over the top level's; a key the frame lacks comes from the top level.  The
    principal point is normalised by the frame's own size, and the images sit in one ragged table."""
    top = dict(CAMS[0], aabb_scale=2)
    frames = [dict(), dict(CAMS[1]), dict(fl_x=22.0, fl_y=21.0, cx=2.5, cy=6.5)]       # frame 2: top-level w, h
    ds = D.NerfDataset(write_capture(str(tmp_path), frames, top), 64, per_frame_cameras=True)
    assert ds.frame_cameras and ds.n_images == 3 and ds.aabb_scale == 2
    assert ds.resolutions.tolist() == [[12, 8], [8, 12], [12, 8]] and ds.resolutions.dtype == torch.int32
    assert ds.pixel_offsets.tolist() == [0, 96, 192, 288] and ds.total_pixels == 288
    assert np.allclose(ds.focal_lengths.numpy(), [[11, 11.5], [9, 9], [22, 21]])
    want_c = np.array([[6 / 12, 4 / 8], [4.25 / 8, 5.5 / 12], [2.5 / 12, 6.5 / 8]], np.float32)
    assert np.array_equal(ds.principal.numpy(), want_c) and np.array_equal(ds.metadata[:, 4:6].numpy(), want_c)
    assert ds.image_data.shape == (288, 4) and ds.shuffle_index.shape == (288,)
    assert [ds.image_resolution(i) for i in range(3)] == [(12, 8), (8, 12), (12, 8)] and ds.resolution == [12, 8]
    assert ds.distortion is None and not hasattr(ds, "focal_eff")
    # the keyword off reads the top level only, as the reference does: frames of one size train with the top-level camera
    off = D.NerfDataset(write_capture(str(tmp_path / "same"), [frames[0], frames[2]], top), 64)
    assert not off.frame_cameras and np.allclose(off.focal_lengths.numpy(), [[11, 11.5]] * 2)


def test_camera_angle_x_resolves_per_frame(tmp_path, fops):
    """A frame's camera_angle_x gives its focal length at the frame's own width, and it overrides a top-level fl_x of that axis; a frame
    with only camera_angle_y keeps the top level's fl_x, as every axis the frame does not name comes from the top level."""
    top = dict(w=12, h=8, fl_x=11.0)
    frames = [dict(), dict(w=8, h=12, camera_angle_x=0.9), dict(camera_angle_y=0.7)]
    ds = D.NerfDataset(write_capture(str(tmp_path), frames, top), 64, per_frame_cameras=True)
    fx1 = D.fov_to_focal_length(8, 0.9 * 180 / math.pi)
    fy2 = D.fov_to_focal_length(8, 0.7 * 180 / math.pi)
    want = np.array([[11, 11], [fx1, fx1], [11, fy2]], np.float32)
    assert np.array_equal(ds.focal_lengths.numpy(), want)


def test_a_frame_without_focal_length_is_named(tmp_path, fops):
    frames = [dict(CAMS[0]), dict(w=12, h=8, cx=4.0)]
    write_capture(str(tmp_path), frames)
    with pytest.raises(RuntimeError, match="images/f1"):
        D.NerfDataset(str(tmp_path), 64, per_frame_cameras=True)
    with pytest.raises(RuntimeError, match="Couldn't read fov"):                      # keyword off: the top level has none either
        D.NerfDataset(str(tmp_path), 64)


def test_a_frame_whose_image_has_another_size_is_refused(tmp_path, fops):
    write_capture(str(tmp_path), [dict(CAMS[0]), dict(CAMS[1])])
    p = os.path.join(str(tmp_path), "transforms_train.json")
    jd = json.load(open(p))
    jd["frames"][1]["w"] = 9
    json.dump(jd, open(p, "w"))
    with pytest.raises(ValueError, match=r"images/f1.*8x12 pixels but its camera is 9x12"):
        D.NerfDataset(str(tmp_path), 64, per_frame_cameras=True)


@pytest.mark.parametrize("extra, err", [(dict(k3=0.01), NotImplementedError), (dict(k4=-0.002), NotImplementedError),
                                        (dict(is_fisheye=True), NotImplementedError), (dict(camera_model="OPENCV_FISHEYE"), NotImplementedError),
                                        (dict(k1=-0.6, k2=0.0), ValueError)])
def test_lens_refusals_fire_per_frame(tmp_path, fops, extra, err):
    """With undistort, the lens refusals apply to every frame on its own -- a refused key in one frame names it -- and check_lens runs at
    the frame's own size (k1 = -0.6 folds over inside the zoomed-out portrait frame)."""
    frames = [dict(CAMS[0], **LENS), dict(CAMS[1], **{**LENS, **extra}), dict(CAMS[2])]
    write_capture(str(tmp_path), frames)
    with pytest.raises(err, match="images/f1"):
        D.NerfDataset(str(tmp_path), 64, per_frame_cameras=True, undistort=True)
    ds = D.NerfDataset(str(tmp_path), 64, per_frame_cameras=True)                      # no undistort: the lens keys are not read
    assert ds.distortion is None and ds.frame_cameras


def test_per_frame_lens(tmp_path, fops):
    frames = [dict(CAMS[0], **LENS), dict(CAMS[1]), dict(CAMS[2], k1=-0.05)]
    ds = D.NerfDataset(write_capture(str(tmp_path), frames), 64, per_frame_cameras=True, undistort=True)
    want = np.array([[0.08, -0.02, 0.003, -0.002], [0, 0, 0, 0], [-0.05, 0, 0, 0]], np.float32)
    assert np.array_equal(ds.distortion.numpy(), want) and np.array_equal(ds.metadata[:, 0:4].numpy(), want)


def fox_small(tmp_path):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_fox_small import materialise
    return materialise(str(tmp_path / "fox"))


DS_TENSORS = ("metadata", "focal_lengths", "principal", "transforms_gpu", "image_data", "shuffle_index")


@pytest.mark.parametrize("undistort", [False, True])
def test_one_camera_loads_exactly_as_the_keyword_off(tmp_path, fops, undistort):
    """fox_small has no per-frame keys: per_frame_cameras=True gives the dataset of the keyword off, tensor for tensor, and the same rays.
    The same holds when every frame repeats the top-level camera in its own keys."""
    root = fox_small(tmp_path)
    for step in range(2):
        on = D.NerfDataset(root, 256, per_frame_cameras=True, undistort=undistort)
        off = D.NerfDataset(root, 256, undistort=undistort)
        assert not on.frame_cameras and on.resolution == off.resolution and on.n_images == off.n_images == 50
        for k in DS_TENSORS + (("distortion", "focal_eff") if undistort else ()):
            a, b = getattr(on, k), getattr(off, k)
            assert a.dtype == b.dtype and torch.equal(a, b), k
        assert not hasattr(on, "frame_extents")
        fops.calls.clear()
        assert all(torch.equal(a, b) for a, b in zip(next(on), next(off)))
        assert fops.calls == ["raygen", "raygen"]
        p = os.path.join(root, "transforms_train.json")
        jd = json.load(open(p))
        keys = {k: jd[k] for k in ("fl_x", "fl_y", "cx", "cy", "w", "h", "k1", "k2", "p1", "p2")}
        for fr in jd["frames"]:
            fr.update(keys)
        json.dump(jd, open(p, "w"))


def mixed(tmp_path, n=7, lens=False, **kw):
    frames = [dict(CAMS[0], **(LENS if lens else {})), dict(CAMS[1]), dict(CAMS[2], **(dict(k1=-0.05) if lens else {}))]
    return D.NerfDataset(write_capture(str(tmp_path), frames, n=n), 64, per_frame_cameras=True, undistort=lens, **kw)


@pytest.mark.parametrize("lens", [False, True])
def test_pixel_ids_map_to_their_frame_pixel_and_ray(tmp_path, fops, lens):
    """Every global pixel id of a mixed capture names the pixel image_pixels gives it, its RGBA is that image's pixel in the file, and
    its ray (the dataset's host tensors through frame_rays) is the fp64 ray through that pixel's centre of that frame's own camera,
    computed from the frame's json keys."""
    from PIL import Image
    ds = mixed(tmp_path, lens=lens)
    jd = json.load(open(os.path.join(str(tmp_path), "transforms_train.json")))
    seen = torch.zeros(ds.total_pixels, dtype=torch.int32)
    for i, fr in enumerate(jd["frames"]):
        w, h = fr["w"], fr["h"]
        pix = ds.image_pixels(i)
        seen[pix.long()] += 1
        im = np.asarray(Image.open(os.path.join(str(tmp_path), fr["file_path"] + ".png")))
        assert np.array_equal(ds.image_data[pix.long()].numpy(), im.reshape(-1, 4))
        ids, o, d = ds.rays_for(pix)
        assert (ids == i).all()
        v, u = np.meshgrid(np.arange(h) + 0.5, np.arange(w) + 0.5, indexing="ij")
        x, y = D.lens_undistort((u.ravel() - fr["cx"]) / fr["fl_x"], (v.ravel() - fr["cy"]) / fr["fl_y"],
                                tuple(fr.get(k, 0.0) for k in D.LENS_KEYS)) if lens else ((u.ravel() - fr["cx"]) / fr["fl_x"],
                                                                                           (v.ravel() - fr["cy"]) / fr["fl_y"])
        m = np.asarray(D.matrix_nerf2ngp(fr["transform_matrix"], D.NERF_SCALE, [0.5, 0.5, 0.5]), np.float64)     # (3, 4)
        want = (m[:, :3] @ np.stack([x, y, np.ones_like(x)])).T
        want /= np.linalg.norm(want, axis=1, keepdims=True)
        assert np.abs(d.double().numpy() - want).max() < 2e-6
        assert np.allclose(o.numpy(), m[:, 3][None].astype(np.float32))
    assert (seen == 1).all()
    assert fops.calls == ["raygen_cams"] * ds.n_images


def test_one_epoch_of_the_ragged_shuffle_visits_every_pixel_once(tmp_path, fops):
    ds = mixed(tmp_path)
    assert torch.equal(ds.shuffle_index.sort().values, torch.arange(ds.total_pixels, dtype=torch.int32))
    n = 37
    drawn = torch.cat([ds.next_pixels(n) for _ in range((ds.total_pixels - 1) // n)])
    rest = ds.shuffle_index[ds.idx_now:]
    assert torch.equal(torch.cat([drawn, rest]).sort().values, torch.arange(ds.total_pixels, dtype=torch.int32))
    again = ds.next_pixels(n)                                                         # past the end: a new permutation of every pixel
    assert ds.idx_now == n and torch.equal(ds.shuffle_index.sort().values, torch.arange(ds.total_pixels, dtype=torch.int32))
    assert torch.equal(again, ds.shuffle_index[:n])


def test_a_split_beyond_int32_pixel_ids_is_refused(tmp_path, fops, monkeypatch):
    monkeypatch.setattr(D, "MAX_PIXELS", 287)
    with pytest.raises(ValueError, match="288 pixels"):
        mixed(tmp_path, n=3)
    monkeypatch.setattr(D, "MAX_PIXELS", 288)
    assert mixed(tmp_path, n=3).total_pixels == 288


@pytest.mark.parametrize("lens", [False, True])
def test_frustum_extents_contain_every_pixel_corner(tmp_path, fops, lens):
    """frame_extents (x_lo, x_hi, y_lo, y_hi) holds the undistorted direction of every pixel corner of its frame (a fixed-point
    iteration, not the dataset's Newton solve) and is tight: the extreme corners lie within 1e-6 of its bounds."""
    ds = mixed(tmp_path, lens=lens)
    jd = json.load(open(os.path.join(str(tmp_path), "transforms_train.json")))
    ext = ds.frame_extents.double().numpy()
    assert ds.frame_extents.shape == (ds.n_images, 4) and ds.frame_extents.dtype == torch.float32
    for i, fr in enumerate(jd["frames"]):
        v, u = np.meshgrid(np.arange(fr["h"] + 1.0), np.arange(fr["w"] + 1.0), indexing="ij")
        xd, yd = (u.ravel() - fr["cx"]) / fr["fl_x"], (v.ravel() - fr["cy"]) / fr["fl_y"]
        x, y = xd.copy(), yd.copy()
        k1, k2, p1, p2 = (fr.get(k, 0.0) for k in D.LENS_KEYS)
        for _ in range(300):
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            x, y = (xd - 2 * p1 * x * y - p2 * (r2 + 2 * x * x)) / rad, (yd - p1 * (r2 + 2 * y * y) - 2 * p2 * x * y) / rad
        lo_x, hi_x, lo_y, hi_y = ext[i]
        assert lo_x <= x.min() and x.max() <= hi_x and lo_y <= y.min() and y.max() <= hi_y, (i, ext[i], x.min(), x.max(), y.min(), y.max())
        assert np.allclose([lo_x, hi_x, lo_y, hi_y], [x.min(), x.max(), y.min(), y.max()], rtol=0, atol=1e-6)
    # an off-centre principal point: the frustum is not symmetric
    assert not np.isclose(-ext[2, 0], ext[2, 1]) and not np.isclose(-ext[2, 2], ext[2, 3])


def test_lens_extent_is_the_symmetric_hull_of_frame_extent():
    W, H, f, c = 1080, 1920, (1375.52, 1374.49), (554.558, 965.268)
    for k in ((0.0578421, -0.0805099, -0.000980296, 0.00015575), (-0.12, 0.02, 0.001, -0.002)):
        lo_x, hi_x, lo_y, hi_y = D.frame_extent(k, W, H, f, c)
        assert D.lens_extent(k, W, H, f, c) == (max(-lo_x, hi_x), max(-lo_y, hi_y))
    assert D.frame_extent(None, W, H, f, c) == (-c[0] / f[0], (W - c[0]) / f[0], -c[1] / f[1], (H - c[1]) / f[1])


def runner_stub(ds, world=1, rank=0, R=32, seed=9):
    return types.SimpleNamespace(dataset={"train": ds}, world_size=world, rank=rank, sampler=types.SimpleNamespace(n_rays_per_batch=R),
                                 _bg_gen=torch.Generator().manual_seed(seed))


def grid_calls(ds, mp):
    """The occupancy-grid entry point the step-0 update calls for ds, by name."""
    from jnerf_b200.plugin.sampler import DensityGridSampler
    seen = []

    class Stop(Exception):
        pass

    def rec(name):
        def f(*a):
            seen.append((name, a))
            raise Stop
        return f
    mp.setattr(ops, "grid_mark_untrained", rec("grid_mark_untrained"))
    mp.setattr(ops, "grid_mark_untrained_cams", rec("grid_mark_untrained_cams"))
    me = types.SimpleNamespace(cfg=types.SimpleNamespace(m_training_step=0), density_grid=torch.zeros(8), dataset=ds,
                               image_resolutions=ds.resolution)
    with pytest.raises(Stop):
        DensityGridSampler.update_density_grid_nerf(me, 0.95, 1, 1)
    return seen


def test_routing_uniform_takes_the_existing_entry_points_and_mixed_the_cams_ones(tmp_path, monkeypatch):
    import cpu_backend
    from jnerf_b200 import runner as R
    cpu_backend.install(monkeypatch)
    f = FrameOps().install(monkeypatch)
    uni = D.NerfDataset(write_capture(str(tmp_path / "u"), [dict(CAMS[0])] * 2, dict(CAMS[0]), n=3), 64, per_frame_cameras=True)
    mix = mixed(tmp_path / "m")
    R.Runner._batch(runner_stub(uni), None)
    uni.generate_rays_total_test(0)
    (name, args), = grid_calls(uni, monkeypatch)
    assert f.calls == ["prepare_batch", "raygen"] and name == "grid_mark_untrained" and args[3] == uni.resolution
    f.calls.clear()
    R.Runner._batch(runner_stub(mix), None)
    mix.generate_rays_total_test(1)
    (name, args), = grid_calls(mix, monkeypatch)
    assert f.calls == ["prepare_batch_cams", "raygen_cams"] and name == "grid_mark_untrained_cams" and args[1] is mix.frame_extents
    # the Runner's per-image size and target
    me = types.SimpleNamespace(background_color=[0.0, 0.0, 0.0])
    for i in range(mix.n_images):
        w, h = R.image_resolution(mix, i)
        tar = R.Runner._target_img(me, mix, i)
        assert tar.shape == (h, w, 3) and (w, h) == mix.image_resolution(i)
        rgba = mix.image_data[mix.image_pixels(i).long()].float() / 255
        assert torch.equal(tar.reshape(-1, 3), rgba[:, :3] * rgba[:, 3:])


def test_synthetic_cameras_stand_in(fops):
    """SyntheticNerfDataset(cameras=...) gives image i the camera cameras[i % len(cameras)]; one camera is the plain stand-in exactly."""
    f = D.fov_to_focal_length(16, 0.6911112070083618 * 180 / math.pi)
    plain = D.SyntheticNerfDataset(n_images=3, H=12, W=16, batch_size=64)
    one = D.SyntheticNerfDataset(n_images=3, batch_size=64, cameras=[(16, 12, f, f, 8.0, 6.0)])
    assert not one.frame_cameras
    for k in DS_TENSORS:
        assert torch.equal(getattr(one, k), getattr(plain, k)), k
    cams = [camera_of(c) for c in CAMS]
    ds = D.SyntheticNerfDataset(n_images=4, batch_size=64, cameras=cams)
    assert ds.frame_cameras and ds.resolutions.tolist() == [[12, 8], [8, 12], [12, 8], [12, 8]]
    assert np.allclose(ds.focal_lengths.numpy()[3], [11, 11.5]) and ds.image_data.shape == (ds.total_pixels, 4)
    o, d = ds.generate_rays_total_test(1)
    assert torch.equal(ds.image_data[ds.image_pixels(1).long()], (ds.shade(o, d) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8))
    # images taken through per-frame lenses, and through one lens on frames of one size
    lensed = D.SyntheticNerfDataset(n_images=3, batch_size=64, cameras=[camera_of(CAMS[0], LENS.values()), camera_of(CAMS[1])], undistort=True)
    assert lensed.frame_cameras and np.allclose(lensed.distortion.numpy()[[0, 2]], [list(LENS.values())] * 2)
    o, d = lensed.generate_rays_total_test(2)
    assert torch.equal(lensed.image_data[lensed.image_pixels(2).long()], (lensed.shade(o, d) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8))
    one = D.SyntheticNerfDataset(n_images=2, H=12, W=16, batch_size=64, distortion=(0.05, 0, 0, 0))
    assert one.image_data.shape == (2, 192, 4)


def test_write_synthetic_frames_round_trips_through_nerf_dataset(tmp_path, fops):
    """write_synthetic_frames writes the cameras in the frames only; NerfDataset(per_frame_cameras=True) reads
    back the stand-in's cameras, poses and pixels, with and without a lens per frame."""
    cams = [camera_of(CAMS[0]), camera_of(CAMS[1]), camera_of(CAMS[2], (-0.05, 0.0, 0.0, 0.0))]
    out = D.write_synthetic_frames(str(tmp_path), cams, n_images=20)
    for split, n in (("train", 20), ("test", 2)):
        src = out[split]
        ds = D.NerfDataset(str(tmp_path), 64, mode=split, per_frame_cameras=True, undistort=True)
        assert ds.n_images == src.n_images == n and ds.frame_cameras
        for k in ("resolutions", "pixel_offsets", "focal_lengths", "principal", "transforms_gpu", "image_data"):
            assert torch.equal(getattr(ds, k), getattr(src, k)), (split, k)
        lensed = np.arange(n) % 3 == 2
        assert np.allclose(ds.distortion.numpy()[lensed], [-0.05, 0, 0, 0]) and not ds.distortion[~lensed].any()
    assert "fl_x" not in json.load(open(os.path.join(str(tmp_path), "transforms_train.json")))


def _gloo_worker(rank, world, port, root, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, HERE)
    import cpu_backend
    from jnerf_b200 import runner as R
    torch.set_num_threads(1)
    mp = pytest.MonkeyPatch()
    cpu_backend.install(mp)
    f = FrameOps().install(mp)
    ds = D.NerfDataset(root, 64, per_frame_cameras=True)
    R.Runner._batch(runner_stub(ds, world, rank, R=24), None)                         # two steps: the second reads past the first
    out = R.Runner._batch(runner_stub(ds, world, rank, R=24, seed=11), None)
    got = [None] * world
    dist.all_gather_object(got, [t.numpy() for t in out])
    ret[rank] = dict(calls=list(f.calls), batches=got)
    mp.undo()
    dist.destroy_process_group()


def test_two_gloo_ranks_take_their_shards_of_the_single_rank_ragged_batch(tmp_path, fops):
    """Two gloo ranks of a mixed capture each build their shard of the global ragged batch with the _cams entry point; side by side the
    shards are the single-rank batch of twice the rays, ray for ray and target for target."""
    import torch.multiprocessing as tmp_mp
    import cpu_backend
    from jnerf_b200 import runner as R
    root = str(tmp_path / "cap")
    frames = [dict(CAMS[0]), dict(CAMS[1]), dict(CAMS[2])]
    write_capture(root, frames, n=7)
    mgr = tmp_mp.Manager()
    ret = mgr.dict()
    tmp_mp.spawn(_gloo_worker, args=(2, 29611 + os.getpid() % 1000, root, ret), nprocs=2, join=True)
    mp = pytest.MonkeyPatch()
    cpu_backend.install(mp)
    try:
        ds = D.NerfDataset(root, 64, per_frame_cameras=True)
        R.Runner._batch(runner_stub(ds, R=48), None)
        single = R.Runner._batch(runner_stub(ds, R=48, seed=11), None)
    finally:
        mp.undo()
    for rank in range(2):
        assert ret[rank]["calls"] == ["prepare_batch_cams"] * 2
        assert all(np.array_equal(a, b) for a, b in zip(ret[rank]["batches"][0], ret[0]["batches"][0]))   # every rank saw the same
    shards = ret[0]["batches"]
    for k, t in enumerate(single):
        assert np.array_equal(np.concatenate([shards[0][k], shards[1][k]]), t.numpy()), k
