"""N2 (SURVEY.md 8f): dataset file parsing and the synthetic stand-ins, without a GPU.  NerfDataset mirrors dataset/dataset.py:68-170
(json discovery by mode, frame skipping, intrinsics, aabb, NeRF -> NGP pose convention, Eigen column-major pose storage);
ray generation itself is a CUDA kernel (ngp_raygen / ngp_prepare_batch) and is checked against the oracle in test_gpu_ops.py."""
import json
import math
import os

import numpy as np
import pytest
import torch

from jnerf_b200.plugin import dataset as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FOX_JSON = os.path.join(GOLDEN, "fox_transforms_train.json")       # data/fox/transforms_train.json of the reference capture, as shipped
FOX_FRAMES = os.path.join(GOLDEN, "fox_small", "frames")            # the frames of that capture that exist on disk (reduced 6x)


@pytest.fixture()
def cpu_device(monkeypatch):
    monkeypatch.setattr(D, "DEVICE", "cpu")


def ref_nerf2ngp(m, scale=0.33, offset=(0.5, 0.5, 0.5), correct_pose=(1, -1, -1)):
    """dataset.py:255-262 restated with numpy."""
    m = np.array(m, np.float32)[:-1, :].copy()
    for k in range(3):
        m[:, k] *= correct_pose[k]
    m[:, 3] = m[:, 3] * scale + np.asarray(offset, np.float32)
    return m[[1, 2, 0]]


def check_against_json(ds, jd, root, n_expected):
    assert ds.n_images == n_expected
    assert ds.resolution == [int(jd["w"]), int(jd["h"])]
    fx = jd["fl_x"] if "fl_x" in jd else 0.5 * ds.W / math.tan(0.5 * jd["camera_angle_x"])
    fy = jd["fl_y"] if "fl_y" in jd else fx
    assert np.allclose(ds.focal_lengths.numpy(), [[fx, fy]] * n_expected)
    assert np.allclose(ds.principal.numpy(), [[jd.get("cx", ds.W / 2) / ds.W, jd.get("cy", ds.H / 2) / ds.H]] * n_expected)
    assert ds.aabb_scale == jd.get("aabb_scale", 1) and ds.aabb_range == (0.5 - ds.aabb_scale / 2, 0.5 + ds.aabb_scale / 2)
    frames = [f for f in jd["frames"] if os.path.exists(os.path.join(root, f["file_path"])) or os.path.exists(os.path.join(root, f["file_path"]) + ".png")]
    xf = ds.transforms_gpu.numpy().reshape(n_expected, 4, 3).transpose(0, 2, 1)        # stored column-major (dataset.py:164-165)
    for k in (0, n_expected // 2, n_expected - 1):
        assert np.array_equal(xf[k], ref_nerf2ngp(frames[k]["transform_matrix"]))
    assert ds.image_data.shape == (n_expected, ds.H * ds.W, 4) and ds.image_data.dtype == torch.uint8


def test_blender_style_dataset(tmp_path, cpu_device):
    """NeRF-synthetic layout (what data/lego looks like): transforms_{train,val,test}.json, camera_angle_x only, RGBA PNGs addressed
    without extension; `train` also takes the val frames (dataset.py:77), `val` mode keeps every 10th frame (:98-99)."""
    from PIL import Image
    rng = np.random.default_rng(0)
    H = W = 16

    def write(split, n):
        os.makedirs(tmp_path / split, exist_ok=True)
        frames = []
        for k in range(n):
            Image.fromarray(rng.integers(0, 256, (H, W, 4), dtype=np.uint8), "RGBA").save(tmp_path / split / f"r_{k}.png")
            m = np.eye(4)
            m[:3, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0]
            m[:3, 3] = rng.standard_normal(3) * 4
            frames.append({"file_path": f"./{split}/r_{k}", "transform_matrix": m.tolist()})
        frames.append({"file_path": f"./{split}/missing", "transform_matrix": np.eye(4).tolist()})        # skipped
        json.dump({"camera_angle_x": 0.6911112070083618, "frames": frames}, open(tmp_path / f"transforms_{split}.json", "w"))
        return frames
    ftrain, fval, ftest = write("train", 5), write("val", 21), write("test", 3)
    tr = D.NerfDataset(str(tmp_path), 64, mode="train")
    assert tr.n_images == 5 + 21 and tr.resolution == [16, 16] and tr.aabb_scale == 1
    fx = 0.5 * 16 / math.tan(0.5 * 0.6911112070083618)
    assert np.allclose(tr.focal_lengths.numpy(), fx) and np.allclose(tr.principal.numpy(), 0.5)
    va = D.NerfDataset(str(tmp_path), 64, mode="val", preload_shuffle=False)
    assert va.n_images == 3                                  # frames[::10] of 22 listed -> 0, 10, 20 (all on disk)
    te = D.NerfDataset(str(tmp_path), 64, mode="test", preload_shuffle=False)
    assert te.n_images == 3
    xf = te.transforms_gpu.numpy().reshape(3, 4, 3).transpose(0, 2, 1)
    assert np.array_equal(xf[1], ref_nerf2ngp(ftest[1]["transform_matrix"]))
    img = np.asarray(Image.open(tmp_path / "test" / "r_1.png"))
    assert np.array_equal(te.image_data[1].numpy().reshape(H, W, 4), img)
    with pytest.raises(AssertionError, match="dataset is not found"):
        D.NerfDataset(str(tmp_path / "train"), 64, mode="train")


def test_fox_stand_in_has_the_captures_numbers():
    """SyntheticNerfDataset(style='fox') takes its resolution / intrinsics / aabb / frame count from data/fox (BASELINE config #3)."""
    F = D.SyntheticNerfDataset.FOX
    jd = json.load(open(FOX_JSON))
    assert (F["W"], F["H"]) == (int(jd["w"]), int(jd["h"])) and F["fl"] == (jd["fl_x"], jd["fl_y"]) and F["c"] == (jd["cx"], jd["cy"])
    assert F["aabb_scale"] == jd["aabb_scale"]
    on_disk = [f for f in jd["frames"] if os.path.exists(os.path.join(FOX_FRAMES, os.path.basename(f["file_path"])))]
    assert F["n_images"] == len(on_disk)
    dist = np.mean([np.linalg.norm(np.array(f["transform_matrix"])[:3, 3]) for f in jd["frames"]])
    assert abs(F["radius"] - dist) < 0.05
    cams = D.synthetic_cameras(16, radius=F["radius"], azimuth=F["azimuth"], elevation=F["elevation"])
    for m in cams:
        pos = m[:3, 3]
        assert abs(np.linalg.norm(pos) - F["radius"]) < 1e-9
        assert np.allclose(-m[:3, 2], -pos / np.linalg.norm(pos))                                      # looks at the origin
        ngp = D.matrix_nerf2ngp(m, D.NERF_SCALE, [0.5, 0.5, 0.5])[:, 3]
        assert np.linalg.norm(ngp - 0.5) < F["backdrop_radius"] and (ngp > -1.5).all() and (ngp < 2.5).all()   # inside backdrop and aabb


def test_fox_stand_in_shading_is_opaque_and_textured():
    ds = object.__new__(D.SyntheticNerfDataset)
    F = D.SyntheticNerfDataset.FOX
    ds.scale, ds.obj_scale, ds.backdrop_radius = D.NERF_SCALE, F["obj_scale"], F["backdrop_radius"]
    m = D.matrix_nerf2ngp(D.synthetic_cameras(1, radius=F["radius"], azimuth=F["azimuth"], elevation=F["elevation"])[0], D.NERF_SCALE, [0.5] * 3)
    H, W = 64, 36
    k = W / F["W"]
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d = np.stack([(u - F["c"][0] * k) / (F["fl"][0] * k), (v - F["c"][1] * H / F["H"]) / (F["fl"][1] * H / F["H"]), np.ones_like(u)], -1).reshape(-1, 3) @ m[:, :3].T
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = np.broadcast_to(m[:, 3], d.shape).copy()
    rgba = ds.shade(torch.from_numpy(o.astype(np.float32)), torch.from_numpy(d.astype(np.float32)))
    assert rgba.shape == (H * W, 4) and bool((rgba[:, 3] == 1).all())                                   # opaque everywhere, like a JPEG frame
    assert float(rgba[:, :3].std()) > 0.1 and 0.1 < float(rgba[:, :3].mean()) < 0.8 and bool(torch.isfinite(rgba).all())
    ds.obj_scale, ds.backdrop_radius = 1.0, None                                                        # lego style: transparent background
    rgba = ds.shade(torch.from_numpy(o.astype(np.float32)), torch.from_numpy(d.astype(np.float32)))
    assert 0.0 < float(rgba[:, 3].mean()) < 1.0


def _cpu_rays_for(self, pix):
    """dataset.py:172-188 restated with torch on the CPU (the product path is the CUDA kernel ngp_raygen)."""
    pix = pix.long()
    img_id = pix // (self.H * self.W)
    off = pix % (self.H * self.W)
    x = ((off % self.W).float() + 0.5) / self.W
    y = ((off // self.W).float() + 0.5) / self.H
    xy = torch.stack([x, y], -1)
    res = torch.tensor([self.W, self.H], dtype=torch.float32)
    d = torch.cat([(xy - self.principal[img_id]) * res / self.focal_lengths[img_id], torch.ones(len(pix), 1)], -1)
    xf = self.transforms_gpu[img_id].reshape(-1, 4, 3).transpose(1, 2)              # back to (3,4)
    d = torch.nn.functional.normalize((xf[:, :, :3] @ d[:, :, None])[:, :, 0], dim=-1)
    return img_id.int(), xf[:, :, 3].contiguous(), d.contiguous()


@pytest.mark.parametrize("style", ["lego", "fox"])
def test_synthetic_datasets_construct_and_render(cpu_device, monkeypatch, style):
    """Both stand-ins build end to end (camera poses, intrinsics, analytic renderer) with the ray generator swapped for its CPU
    restatement: the lego style has a transparent background, the fox style is opaque, and every camera sees the objects."""
    monkeypatch.setattr(D._RayBatcher, "rays_for", _cpu_rays_for)
    kw = dict(n_images=3, H=48, W=27) if style == "fox" else dict(n_images=3, H=32, W=32)
    ds = D.SyntheticNerfDataset(batch_size=64, mode="train", style=style, seed=1, **kw)
    assert ds.n_images == 3 and ds.resolution == [kw["W"], kw["H"]]
    assert ds.image_data.shape == (3, kw["H"] * kw["W"], 4) and ds.image_data.dtype == torch.uint8
    a = ds.image_data[:, :, 3].float() / 255
    if style == "fox":
        assert ds.aabb_scale == 4 and ds.aabb_range == (-1.5, 2.5) and bool((a == 1).all())
        F = D.SyntheticNerfDataset.FOX
        assert abs(ds._focal[0] - F["fl"][0] * 27 / F["W"]) < 1e-6 and abs(ds._cy - F["c"][1] * 48 / F["H"]) < 1e-6
    else:
        assert ds.aabb_scale == 1 and ds.aabb_range == (0.0, 1.0) and 0.05 < float(a.mean()) < 0.95
    for k in range(3):
        assert float(ds.image_data[k, :, :3].float().std()) > 5.0                    # every view shows structure
    img_ids, o, d, rgba = next(ds)
    assert o.shape == (64, 3) and d.shape == (64, 3) and rgba.shape == (64, 4) and float(rgba.max()) <= 1.0
    assert torch.allclose(d.norm(dim=-1), torch.ones(64), atol=1e-5)
    val = D.SyntheticNerfDataset(batch_size=64, mode="val", style=style, seed=1, **dict(kw, n_images=20))
    assert val.n_images == 2                                                        # a tenth of the views, other cameras than training


def test_reduced_fox_capture_fixture(tmp_path, cpu_device):
    """tests/golden/fox_small: the reference's data/fox reduced 6x (make_fox_small.py), materialised in the reference's dataset layout
    and read by NerfDataset -- the real-capture input of the GPU end-to-end test."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_fox_small import materialise
    root = materialise(str(tmp_path / "fox"))
    jd = json.load(open(os.path.join(root, "transforms_train.json")))
    assert len(jd["frames"]) == 67                                   # 17 of them have no image: skipped by the loader
    ds = D.NerfDataset(root, 4096, mode="train")
    check_against_json(ds, jd, root, 50)
    assert ds.resolution == [180, 320] and ds.aabb_scale == 4 and bool((ds.image_data[:, :, 3] == 255).all())
    assert D.NerfDataset(root, 4096, mode="test", preload_shuffle=False).n_images == 2
    rj = json.load(open(FOX_JSON))                                   # same poses as the capture, intrinsics scaled by the reduction
    assert [f["file_path"] for f in rj["frames"]] == [f["file_path"] for f in jd["frames"]]
    assert np.array_equal(np.array([f["transform_matrix"] for f in rj["frames"]]), np.array([f["transform_matrix"] for f in jd["frames"]]))
    for k in ("fl_x", "fl_y", "cx", "cy"):
        assert abs(jd[k] * 6 - rj[k]) < 1e-9
    assert jd["aabb_scale"] == rj["aabb_scale"] and (jd["w"], jd["h"]) == (rj["w"] // 6, rj["h"] // 6)
    assert float(ds.image_data[:, :, :3].float().std()) > 20         # photographs, not blanks
