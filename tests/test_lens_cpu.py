"""Lens distortion of Instant-NGP captures (`undistort=True`), without a GPU: reading k1, k2, p1, p2 per split, what the radial-tangential
model refuses, the fp64 fold check, the effective focal lengths of the occupancy grid's visibility frustum, and that every ray batch the
datasets and the Runner build -- on every data-parallel rank -- is handed the lens, while `undistort=False` hands over exactly what it did
before.  The lens kernels themselves are checked on the GPU (test_lens_gpu.py)."""
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
FOX_LENS = (0.0578421, -0.0805099, -0.000980296, 0.00015575)          # data/fox/transforms_train.json


@pytest.fixture()
def cpu_device(monkeypatch):
    monkeypatch.setattr(D, "DEVICE", "cpu")


def lens_rays(pix, W, H, xforms, focal, principal, distortion=None):
    """The rays of ngp_raygen / ngp_raygen_lens restated in fp64: every pixel's normalised coordinate undistorted by a fixed-point
    iteration (not the kernels' Newton solve), the direction through the camera's axes, normalised."""
    pix = pix.long().numpy()
    n_img = xforms.shape[0]
    ids, off = pix // (H * W), pix % (H * W)
    m = xforms.double().numpy().reshape(n_img, 4, 3)[ids]                          # rows: camera x, y, z axes, origin
    xd = ((off % W) + 0.5 - principal[ids, 0].double().numpy() * W) / focal[ids, 0].double().numpy()
    yd = ((off // W) + 0.5 - principal[ids, 1].double().numpy() * H) / focal[ids, 1].double().numpy()
    x, y = xd.copy(), yd.copy()
    if distortion is not None:
        k1, k2, p1, p2 = distortion.double().numpy()[ids].T
        for _ in range(200):
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            x = (xd - 2 * p1 * x * y - p2 * (r2 + 2 * x * x)) / rad
            y = (yd - p1 * (r2 + 2 * y * y) - 2 * p2 * x * y) / rad
    d = m[:, 0] * x[:, None] + m[:, 1] * y[:, None] + m[:, 2]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return torch.from_numpy(ids.astype(np.int32)), torch.from_numpy(m[:, 3].astype(np.float32)), torch.from_numpy(d.astype(np.float32))


class LensOps:
    """CPU stand-ins of ops.raygen / ops.prepare_batch that accept the lens and record what every call was handed."""

    def __init__(self):
        self.calls = []

    def raygen(self, pix, W, H, xforms, focal, principal, **kw):
        self.calls.append(("raygen", kw.get("distortion")))
        return lens_rays(pix, W, H, xforms, focal, principal, ops.lens_of(kw.get("distortion")))

    def prepare_batch(self, pix, W, H, xforms, focal, principal, images, bg, **kw):
        self.calls.append(("prepare_batch", kw.get("distortion")))
        img, o, d = lens_rays(pix, W, H, xforms, focal, principal, ops.lens_of(kw.get("distortion")))
        rgba = images.reshape(-1, 4)[pix.long()].float() / 255.0
        return img, o, d, rgba[:, :3] * rgba[:, 3:] + bg * (1 - rgba[:, 3:])


@pytest.fixture()
def lens_ops(monkeypatch, cpu_device):
    fake = LensOps()
    monkeypatch.setattr(ops, "raygen", fake.raygen)
    monkeypatch.setattr(ops, "prepare_batch", fake.prepare_batch)
    return fake


def fox_small(tmp_path):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_fox_small import materialise
    return materialise(str(tmp_path / "fox"))


def edit_json(root, split, **kv):
    p = os.path.join(root, f"transforms_{split}.json")
    jd = json.load(open(p))
    for k, v in kv.items():
        if v is None:
            jd.pop(k, None)
        else:
            jd[k] = v
    json.dump(jd, open(p, "w"))


def test_fox_small_lens_is_read_per_split(tmp_path, lens_ops):
    """Each split takes k1, k2, p1, p2 from its own json into metadata[:, 0:4] (the reference's slots) and ds.distortion; the rest of the
    metadata is what undistort=False gives."""
    root = fox_small(tmp_path)
    other = (0.01, -0.02, 0.003, -0.004)
    edit_json(root, "test", **dict(zip(D.LENS_KEYS, other)))
    for split, lens, n in (("train", FOX_LENS, 50), ("test", other, 2)):
        on = D.NerfDataset(root, 4096, mode=split, undistort=True)
        off = D.NerfDataset(root, 4096, mode=split)
        want = np.tile(np.array(lens, np.float32), (n, 1))
        assert np.array_equal(on.metadata[:, 0:4].numpy(), want) and np.array_equal(on.distortion.numpy(), want)
        assert on.distortion.shape == (n, 4) and on.distortion.dtype == torch.float32
        assert np.array_equal(on.metadata[:, 4:].numpy(), off.metadata[:, 4:].numpy())
        assert np.array_equal(on.principal.numpy(), off.principal.numpy()) and np.array_equal(on.focal_lengths.numpy(), off.focal_lengths.numpy())


def test_undistort_off_hands_the_kernels_what_it_did_before(tmp_path, lens_ops):
    """undistort=False: metadata[:, 0:4] stays 0, there is no lens and no effective focal length, and every ray call is the pinhole call
    of the parent (no distortion argument at all)."""
    root = fox_small(tmp_path)
    ds = D.NerfDataset(root, 256, mode="train")
    assert not ds.metadata[:, 0:4].any() and ds.distortion is None and not hasattr(ds, "focal_eff")
    next(ds)
    ds.generate_rays_total_test(1)
    assert lens_ops.calls == [("raygen", None), ("raygen", None)]
    lens_ops.calls.clear()
    on = D.NerfDataset(root, 256, mode="train", undistort=True)
    next(on)
    on.generate_rays_total_test(1)
    assert [c[0] for c in lens_ops.calls] == ["raygen", "raygen"] and all(c[1] is on.distortion for c in lens_ops.calls)


def test_missing_coefficients_count_as_zero(tmp_path, lens_ops):
    root = fox_small(tmp_path)
    edit_json(root, "test", k1=None, k2=None, p1=0.002, p2=None)
    ds = D.NerfDataset(root, 4096, mode="test", undistort=True)
    assert np.array_equal(ds.distortion.numpy(), np.tile(np.array([0, 0, 0.002, 0], np.float32), (2, 1)))
    edit_json(root, "test", p1=None)
    ds = D.NerfDataset(root, 4096, mode="test", undistort=True)
    assert not ds.distortion.any() and not hasattr(ds, "focal_eff")
    assert ops.lens_of(ds.distortion) is None                                     # a lens of zeros takes the pinhole kernels


@pytest.mark.parametrize("extra", [dict(k3=0.01), dict(k4=-0.002), dict(is_fisheye=True), dict(camera_model="OPENCV_FISHEYE")])
def test_models_the_kernels_cannot_represent_are_refused(tmp_path, lens_ops, extra):
    root = fox_small(tmp_path)
    edit_json(root, "test", **extra)
    with pytest.raises(NotImplementedError):
        D.NerfDataset(root, 4096, mode="test", undistort=True)
    assert D.NerfDataset(root, 4096, mode="test").n_images == 2                   # undistort=False reads the json as before
    edit_json(root, "test", **{k: None for k in extra})
    if "k3" in extra:
        edit_json(root, "test", k3=0.0)                                           # a zero k3 is the model
        assert D.NerfDataset(root, 4096, mode="test", undistort=True).n_images == 2


def test_a_lens_that_folds_over_inside_the_image_is_refused(tmp_path, lens_ops):
    """k1 = -0.3 at the fox capture's field of view: r (1 + k1 r^2) turns back (1 + 3 k1 r^2 = 0 at r = 1.05) before it reaches the
    farthest corner (r_d = 0.81), so two directions share pixels.  A strong but invertible lens (k1 = 0.25) loads."""
    root = fox_small(tmp_path)
    edit_json(root, "test", k1=-0.3, k2=0.0, p1=0.0, p2=0.0)
    with pytest.raises(ValueError, match=r"k1 = -0\.3.*folds over"):
        D.NerfDataset(root, 4096, mode="test", undistort=True)
    edit_json(root, "test", k1=0.25)
    assert D.NerfDataset(root, 4096, mode="test", undistort=True).n_images == 2
    with pytest.raises(ValueError, match="k1 = -0.3"):
        D.SyntheticNerfDataset(style="fox", H=64, W=36, n_images=2, distortion=(-0.3, 0, 0, 0))


def test_fold_check_against_the_radial_closed_form():
    """For a radial lens k1 < 0, r (1 + k1 r^2) folds at r^2 = -1 / (3 k1) with the largest distorted radius 2/3 r there: the check
    refuses exactly the lenses whose largest distorted radius is below the farthest corner's."""
    W, H, f, c = 1080, 1920, (1375.52, 1374.49), (554.558, 965.268)
    reach = math.hypot(max(c[0], W - c[0]) / f[0], max(c[1], H - c[1]) / f[1])
    k_crit = -4 / (27 * reach * reach)                                           # (2/3) r_fold = reach
    D.check_lens((k_crit * 0.97, 0, 0, 0), W, H, f, c)
    with pytest.raises(ValueError):
        D.check_lens((k_crit * 1.03, 0, 0, 0), W, H, f, c)


def test_effective_focal_lengths_hold_the_undistorted_extent(tmp_path, lens_ops):
    """focal_eff = (W/2) / max|x_u|, (H/2) / max|y_u| over the fp64 undistorted coordinates of ALL pixel centres and corners."""
    root = fox_small(tmp_path)
    for lens in (FOX_LENS, (-0.12, 0.02, 0.001, -0.002)):
        edit_json(root, "train", **dict(zip(D.LENS_KEYS, lens)))
        ds = D.NerfDataset(root, 4096, mode="train", undistort=True)
        W, H = ds.resolution
        fx, fy = ds._focal
        u, v = np.meshgrid(np.arange(2 * W + 1) / 2, np.arange(2 * H + 1) / 2)     # corners (integers) and centres (halves)
        xd, yd = (u - ds._cx) / fx, (v - ds._cy) / fy
        # the fixed-point restatement of lens_rays, on every centre and corner
        x, y = xd.copy(), yd.copy()
        k1, k2, p1, p2 = lens
        for _ in range(200):
            r2 = x * x + y * y
            rad = 1 + r2 * (k1 + r2 * k2)
            x, y = (xd - 2 * p1 * x * y - p2 * (r2 + 2 * x * x)) / rad, (yd - p1 * (r2 + 2 * y * y) - 2 * p2 * x * y) / rad
        want = np.array([W / 2 / np.abs(x).max(), H / 2 / np.abs(y).max()])
        got = ds.focal_eff.double().numpy()
        assert got.shape == (50, 2) and np.allclose(got, want[None], rtol=1e-6, atol=0), (got[0], want)


def test_synthetic_capture_through_a_lens(lens_ops):
    """SyntheticNerfDataset(distortion=...) takes its images through the lens whatever `undistort` says; `undistort` decides whether its
    rays go through it too.  Without a lens, the images are the pinhole stand-in's."""
    kw = dict(style="fox", H=48, W=27, n_images=2, batch_size=64)
    lens = (-0.1, 0.02, 0.001, -0.001)
    pin = D.SyntheticNerfDataset(**kw)
    off = D.SyntheticNerfDataset(distortion=lens, **kw)
    on = D.SyntheticNerfDataset(distortion=lens, undistort=True, **kw)
    zero = D.SyntheticNerfDataset(undistort=True, **kw)
    assert torch.equal(off.image_data, on.image_data) and not torch.equal(pin.image_data, on.image_data)
    assert torch.equal(zero.image_data, pin.image_data) and not zero.distortion.any()
    assert off.distortion is None and not off.metadata[:, 0:4].any()
    assert np.allclose(on.distortion.numpy(), np.array([lens] * 2, np.float32)) and hasattr(on, "focal_eff")
    # the pixels' colours are the scene along the undistorted rays
    o, d = on.generate_rays_total_test(0)
    assert torch.equal(on.image_data[0], (on.shade(o, d) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8))


def test_fox_cfg_sets_undistort_in_every_split():
    from jnerf_b200.runner import fox_cfg
    on, off = fox_cfg(undistort=True), fox_cfg()
    assert all(s["undistort"] is True for s in on["dataset"].values())
    assert all("undistort" not in s for s in off["dataset"].values())
    assert on["dataset"]["train"] == dict(off["dataset"]["train"], undistort=True)


def test_runner_batches_hand_every_rank_the_same_lens(monkeypatch):
    """Runner._batch under world_size 2: both ranks build their shard of the same global pixel batch with the dataset's lens, and their
    rays are the lens rays of exactly those pixels."""
    import cpu_backend
    from jnerf_b200 import runner as R
    cpu_backend.install(monkeypatch)                                              # torch's "cuda" is the CPU
    monkeypatch.setattr(D, "DEVICE", "cpu")
    lens_ops = LensOps()
    monkeypatch.setattr(ops, "raygen", lens_ops.raygen)
    monkeypatch.setattr(ops, "prepare_batch", lens_ops.prepare_batch)
    kw = dict(style="fox", H=48, W=27, n_images=3, batch_size=64, distortion=FOX_LENS, undistort=True, seed=4)
    shards, lenses = [], []
    ref = D.SyntheticNerfDataset(**kw)
    pix_all = ref.next_pixels(2 * 32)
    for rank in range(2):
        ds = D.SyntheticNerfDataset(**kw)
        me = types.SimpleNamespace(dataset={"train": ds}, world_size=2, rank=rank, sampler=types.SimpleNamespace(n_rays_per_batch=32),
                                   _bg_gen=torch.Generator().manual_seed(9))
        lens_ops.calls.clear()
        img_ids, rays_o, rays_d, bg, target = R.Runner._batch(me, None)
        (name, lens), = lens_ops.calls
        assert name == "prepare_batch" and lens is ds.distortion
        lenses.append(lens)
        pix = pix_all[rank * 32:(rank + 1) * 32]
        _, _, want = lens_rays(pix, ds.W, ds.H, ds.transforms_gpu, ds.focal_lengths, ds.principal, ds.distortion)
        assert torch.equal(rays_d, want)
        shards.append(rays_d)
    assert torch.equal(lenses[0], lenses[1]) and not torch.equal(shards[0], shards[1])


def test_occupancy_grid_visibility_takes_the_effective_focal_lengths(lens_ops):
    """The step-0 grid update marks cells untrained with focal_eff when the dataset has one, with the focal lengths otherwise."""
    from jnerf_b200.plugin.sampler import DensityGridSampler
    seen = []

    class Stop(Exception):
        pass

    def mark(grid, focal, xforms, res):
        seen.append(focal)
        raise Stop

    for lens in (None, FOX_LENS):
        ds = D.SyntheticNerfDataset(style="fox", H=48, W=27, n_images=2, distortion=lens, undistort=lens is not None)
        me = types.SimpleNamespace(cfg=types.SimpleNamespace(m_training_step=0), density_grid=torch.zeros(8), dataset=ds,
                                   image_resolutions=ds.resolution)
        mp = pytest.MonkeyPatch()
        mp.setattr(ops, "grid_mark_untrained", mark)
        with pytest.raises(Stop):
            DensityGridSampler.update_density_grid_nerf(me, 0.95, 1, 1)
        mp.undo()
    assert seen[0] is not None and torch.equal(seen[0], torch.tensor([[27 * 1375.52 / 1080, 48 * 1374.49 / 1920]] * 2))
    assert seen[1] is not None and not torch.equal(seen[1], seen[0])


def test_lens_of_reads_the_device_once_per_version(monkeypatch):
    """ops.lens_of: None and all-zero lenses select the pinhole entry points; the answer is kept on the tensor and refreshed when it is
    written in place."""
    z = torch.zeros(3, 4)
    assert ops.lens_of(None) is None and ops.lens_of(z) is None
    reads = []
    any_ = torch.Tensor.any
    monkeypatch.setattr(torch.Tensor, "any", lambda self, *a, **k: reads.append(1) or any_(self, *a, **k))
    assert ops.lens_of(z) is None and not reads                                     # kept from the first call
    z[1, 0] = 0.05
    assert ops.lens_of(z) is z and len(reads) == 1
    assert ops.lens_of(z) is z and len(reads) == 1
    # and the entry point follows it
    names = []
    monkeypatch.setattr(ops, "_p", lambda t: 0)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops.lib, "call", lambda name, *a: names.append(name))
    pix = torch.zeros(4, dtype=torch.int32)
    ops.raygen(pix, 2, 2, None, None, None, distortion=z)
    ops.raygen(pix, 2, 2, None, None, None, distortion=torch.zeros(3, 4))
    ops.raygen(pix, 2, 2, None, None, None)
    img = torch.zeros((3, 4, 4), dtype=torch.uint8)
    ops.prepare_batch(pix, 2, 2, None, None, None, img, None, distortion=z)
    ops.prepare_batch(pix, 2, 2, None, None, None, img, None, distortion=torch.zeros(3, 4))
    assert names == ["ngp_raygen_lens", "ngp_raygen", "ngp_raygen", "ngp_prepare_batch_lens", "ngp_prepare_batch"]
