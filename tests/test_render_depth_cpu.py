"""Depth maps and the spiral camera path without a GPU: the C-ABI argument checks of the depth composite, the NGP-to-NeRF unit
conversion and opacity normalisation (depth_from_sum), the depth outputs of Runner.render_depth_with_pose / test / render through a
depth-capable stand-in of ops.render_rays, and utils/camera_path.path_spiral on the forward-facing stand-in."""
import ctypes
import os

import numpy as np
import pytest
import torch

import render_cpu_backend


def install_depth(monkeypatch, fake):
    """tests/render_cpu_backend.py's render_rays plus a `depth` argument.  Its depth is alpha * |o - (0.5, 0.5, 0.5)|: every ray's weights
    put the expected t at its camera's distance from the scene centre, so the normalised depth of a covered pixel is that distance
    in NeRF units (/ scale), whatever the stand-in's network makes of the samples."""
    render_cpu_backend.install(monkeypatch, fake)
    import jnerf_b200.ops as real_ops
    colour = real_ops.render_rays
    seen = []

    def render_rays(rays_o, rays_d, *a, depth=False, **k):
        seen.append(depth)
        rgb, alpha, n, rounds = colour(rays_o, rays_d, *a, **k)
        if not depth:
            return rgb, alpha, n, rounds
        S = alpha[:, 0] * (rays_o.float() - 0.5).norm(dim=1)
        return rgb, alpha, n, rounds, S
    monkeypatch.setattr(real_ops, "render_rays", render_rays)
    return seen


def make(monkeypatch, tmp_path, H=12, W=16, rays=64):
    from test_runner_cpu import make_runner
    r, fake = make_runner(monkeypatch, rays=rays, H=H, W=W, log_dir=str(tmp_path), exp_name="lego_t")
    seen = install_depth(monkeypatch, fake)
    r.cfg.dataset.test.n_images, r.cfg.dataset.test.H, r.cfg.dataset.test.W = 20, H, W
    return r, fake, seen


def test_depth_from_sum_converts_units_and_normalises():
    from jnerf_b200.runner import depth_from_sum
    alpha = torch.tensor([[1.0], [0.5], [0.0], [0.25]])
    t = torch.tensor([1.32, 0.66, 0.9, 0.2])                              # expected t in model units
    S = alpha[:, 0] * t
    for scale in (0.33, 0.05):
        d = depth_from_sum(S, alpha, scale)
        assert d.shape == (4,) and d.dtype == torch.float32
        assert torch.allclose(d[[0, 1, 3]], t[[0, 1, 3]] / scale, rtol=1e-6)
        assert d[2] == 0                                                   # alpha 0: no depth, not a division by zero
    assert depth_from_sum(torch.zeros(3), torch.zeros(3, 1), 0.33).eq(0).all()


@pytest.mark.parametrize("scale", [0.33, 0.05])
def test_render_depth_with_pose_is_in_nerf_units(monkeypatch, tmp_path, scale):
    """The stand-in's cameras sit 4 NeRF units from the origin; with the default scale and a config-set one (0.05, as ngp_comp.py's
    Scarf scene) the covered pixels come out at 4, the empty ones at 0."""
    r, fake, seen = make(monkeypatch, tmp_path)
    ds = r.dataset["train"]
    ds.scale = scale
    img, depth, alpha = r.render_depth_with_pose(ds.poses[1])
    assert img.shape == (12, 16, 3) and depth.shape == (12, 16) and alpha.shape == (12, 16, 1) and seen == [True]
    cam = float(np.linalg.norm(ds.poses[1][:3, 3]))
    assert abs(cam - 4.0) < 1e-5
    a = alpha[..., 0]
    assert (a > 0).any() and ((a == 0).any() or scale < 0.25)           # at 0.05 the camera sits inside the occupied sphere
    assert torch.allclose(depth[a > 0], torch.full_like(depth[a > 0], cam), rtol=1e-5)
    assert (depth[a == 0] == 0).all()
    # the colour image is the one render_img_with_pose gives under the same jitter
    s = r.sampler
    s.rng[:] = rng0 = s.rng.copy()
    img1, _, _ = r.render_depth_with_pose(ds.poses[1])
    s.rng[:] = rng0
    assert torch.equal(img1, r.render_img_with_pose(ds.poses[1]))


def test_render_rays_without_depth_keeps_four_values(monkeypatch, tmp_path):
    r, fake, seen = make(monkeypatch, tmp_path)
    o, d = r.dataset["train"].generate_rays_total_test(0)
    out = r.render_rays(o, d)
    assert len(out) == 4 and seen == [False]
    out = r.render_rays(o, d, depth=True)
    assert len(out) == 5 and out[4].shape == (o.shape[0],) and seen == [False, True]


def test_test_writes_depth_maps_from_the_same_render(monkeypatch, tmp_path, capsys):
    from PIL import Image
    r, fake, seen = make(monkeypatch, tmp_path)
    fake.calls.clear()
    r.test(min_transmittance=0.0, depth=True)
    out = tmp_path / "lego_t" / "test"
    assert sorted(os.listdir(out)) == ["lego_t_depth_0.npy", "lego_t_depth_0.png", "lego_t_depth_1.npy", "lego_t_depth_1.png",
                                       "lego_t_gt_0.png", "lego_t_gt_1.png", "lego_t_r_0.png", "lego_t_r_1.png"]
    assert fake.calls.count("render_rays") == 2 and seen == [True, True]              # one render per view, colour and depth
    for i in range(2):
        dep = np.load(out / f"lego_t_depth_{i}.npy")
        png = np.asarray(Image.open(out / f"lego_t_depth_{i}.png"))
        assert dep.dtype == np.float32 and dep.shape == (12, 16) and png.dtype == np.uint8 and png.shape == (12, 16)
        covered = dep > 0
        assert covered.any() and np.allclose(dep[covered], 4.0, rtol=1e-5)
        assert (png[~covered] == 0).all() and (png[covered] > 0).any()
    # without depth: the files and calls of the colour-only test
    seen.clear()
    r.render_test(save_path=str(tmp_path / "plain"))
    assert seen == [False, False] and not any("depth" in f for f in os.listdir(tmp_path / "plain"))


def test_depth_to_grey_is_brighter_when_nearer():
    from jnerf_b200.runner import depth_to_grey
    depth = torch.tensor([[1.0, 2.0, 3.0, 5.0, 0.0]])
    alpha = torch.tensor([[1.0, 1.0, 1.0, 1.0, 0.0]])
    g = depth_to_grey(depth, alpha, 1.0, 3.0)
    assert g.dtype == np.uint8 and list(g[0]) == [255, 128, 0, 0, 0]
    assert list(depth_to_grey(depth, alpha * 0.5, 1.0, 3.0)[0]) == [128, 64, 0, 0, 0]


def test_render_writes_a_depth_video_beside_the_colour_one(monkeypatch, tmp_path):
    cv2 = pytest.importorskip("cv2")
    r, fake, seen = make(monkeypatch, tmp_path, H=16, W=24, rays=128)
    fake.calls.clear()
    path = r.render(depth=True)
    assert path == os.path.join(str(tmp_path), "lego_t", "demo.mp4")
    dpath = os.path.join(str(tmp_path), "lego_t", "demo_depth.mp4")

    def frames(p):
        cap, out = cv2.VideoCapture(p), []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            out.append(f)
        cap.release()
        return out
    col, dep = frames(path), frames(dpath)
    assert len(col) == len(dep) == 80 and all(f.shape == (16, 24, 3) for f in col + dep)
    assert fake.calls.count("render_rays") == 80 and seen == [True] * 80                  # the depth frames come from the colour renders
    # every camera of the spherical path sits 4 units out: one fixed range gives every covered pixel the same shade in every frame
    lit = np.concatenate([f[..., 0][f[..., 0] > 40] for f in dep])
    assert lit.size > 0 and np.percentile(lit, 90) - np.percentile(lit, 10) <= 24
    # another camera path, without depth: no depth file, one frame a pose
    seen.clear()
    from jnerf_b200.utils.camera_path import path_spherical
    p2 = str(tmp_path / "short.mp4")
    r.render(save_path=p2, poses=path_spherical(5))
    assert len(frames(p2)) == 5 and seen == [False] * 5 and not os.path.exists(str(tmp_path / "short_depth.mp4"))


def test_depth_range_from_bounds_or_the_box(monkeypatch, tmp_path):
    r, fake, seen = make(monkeypatch, tmp_path)
    ds = r.dataset["train"]
    pose = np.eye(4, dtype=np.float32)[:3]
    pose[2, 3] = 4.0                                                      # 4 units out along z, the box is [-1.52, 1.52]^3 in NeRF units
    near, far = r.depth_range([pose])
    h = 0.5 / ds.scale
    assert abs(near - (4.0 - h)) < 1e-4 and abs(far - np.sqrt((4.0 + h) ** 2 + 2 * h * h)) < 1e-4
    ds.bounds = np.array([[1.5, 9.0], [2.0, 7.0]], np.float32)
    assert r.depth_range([pose]) == (1.5, 9.0)


def test_c_abi_rejects_malformed_depth_composite_arguments():
    from jnerf_b200 import lib
    lib.load()
    n = np.zeros(1, np.uint32)
    npp = n.ctypes.data_as(ctypes.c_void_p)
    fake_ws, fake_depth = 1 << 20, 1 << 21                                # never dereferenced: the checks come first

    def composite(capacity, ws, n_alive, k, depth=fake_depth):
        return lib.call("ngp_render_composite_round_depth", None, 10, capacity, ws, n_alive, k, 1e-4, 5, None, None, None, depth, npp)
    with pytest.raises(lib.NgpError, match="depth_out"):
        composite(64, fake_ws, 1, 1, depth=None)
    with pytest.raises(lib.NgpError, match="capacity"):
        composite(0, fake_ws, 1, 1)
    with pytest.raises(lib.NgpError, match="workspace"):
        composite(64, None, 1, 1)
    with pytest.raises(lib.NgpError, match="k_steps"):
        composite(64, fake_ws, 1, 0)
    with pytest.raises(lib.NgpError, match="n_alive"):
        composite(64, fake_ws, 11, 1)
    assert composite(64, fake_ws, 0, 1) == 0 and n[0] == 0               # nothing alive: nothing to do
    assert lib.KERNELS_PER_CALL["ngp_render_composite_round_depth"] == lib.KERNELS_PER_CALL["ngp_render_composite_round"]


# ------------------------------------------------------------------------------------------------ spiral camera path
@pytest.fixture()
def llff(monkeypatch, tmp_path):
    from jnerf_b200.plugin import dataset as D
    monkeypatch.setattr(D, "DEVICE", "cpu")
    D.write_synthetic_llff(str(tmp_path), n_images=9, H=24, W=32, seed=2)
    return D.LLFFDataset(str(tmp_path), 64, mode="train", factor=1, llffhold=4)


def test_llff_dataset_keeps_the_rescaled_bounds(llff, tmp_path):
    arr = np.load(tmp_path / "poses_bounds.npy")
    b = llff.bounds
    assert b.shape == (len(llff.poses), 2) and b.dtype == np.float32
    raw = arr[llff.i_select, -2:]
    sc = 1.0 / (arr[:, -2:].min() * 0.75)                                 # bd_factor 0.75: the nearest bound of the capture becomes 1 / 0.75
    assert np.allclose(b, raw * sc, rtol=1e-6) and abs(arr[:, -2:].min() * sc - 1 / 0.75) < 1e-6


def test_path_spiral_on_the_forward_facing_stand_in(llff):
    from jnerf_b200.utils.camera_path import path_spiral
    poses, bounds = np.stack(llff.poses).astype(np.float64), llff.bounds.astype(np.float64)
    path = path_spiral(llff.poses, llff.bounds)
    assert len(path) == 120 and all(p.shape == (3, 4) and p.dtype == np.float32 for p in path)
    assert len(path_spiral(llff.poses, llff.bounds, n_frames=7)) == 7
    # the average camera and focus point, restated: mean position, summed viewing axis and up vector, focus depth from the bounds
    z = poses[:, :, 2].sum(0)
    z /= np.linalg.norm(z)
    up = poses[:, :, 1].sum(0)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    centre = poses[:, :, 3].mean(0)
    close, inf = 0.9 * bounds.min(), 5.0 * bounds.max()
    focal = 1.0 / (0.25 / close + 0.75 / inf)
    focus = centre - focal * z
    rads = np.percentile(np.abs(poses[:, :, 3]), 90, 0)
    R = np.stack([x, y, z], 1)
    for p in path:
        p = p.astype(np.float64)
        c, view = p[:, 3], -p[:, 2]                                       # the camera looks along -z
        assert abs(np.linalg.det(p[:, :3]) - 1) < 1e-5
        v = focus - c
        miss = np.linalg.norm(v - (v @ view) * view)                      # distance of the focus point from the viewing axis
        assert miss <= 1e-5 * max(1.0, np.linalg.norm(v)) and v @ view > 0
        off = R.T @ (c - centre)                                          # offset from the average camera, in its frame
        assert (np.abs(off) <= rads + 1e-5).all()
    offs = np.stack([R.T @ (p[:, 3].astype(np.float64) - centre) for p in path])
    assert (np.abs(offs[:, :2]).max(0) > 0.9 * rads[:2]).all()            # the spiral spans its radii
    with pytest.raises(ValueError, match="bounds"):
        path_spiral(llff.poses, None)
