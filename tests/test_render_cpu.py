"""Rendering without a GPU: the camera path against hand-computed poses, and the host logic of Runner.render_rays /
render_img_with_pose / render / test through tests/render_cpu_backend.py (rays, jitter stream, files, PSNR), plus the argument checks of
the renderer's C ABI."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import oracle_lib as ol
import render_cpu_backend

S3 = math.sqrt(3.0)


def test_path_spherical_matches_hand_computed_poses():
    from jnerf_b200.utils.camera_path import path_spherical, pose_spherical
    path = path_spherical()
    assert len(path) == 80 and all(p.shape == (3, 4) and p.dtype == np.float32 for p in path)
    # azimuth -180, -90 and 0 degrees at elevation -30, radius 4
    want = {0: [[1, 0, 0, 0], [0, 0.5, -S3 / 2, -2 * S3], [0, S3 / 2, 0.5, 2]],
            20: [[0, 0.5, -S3 / 2, -2 * S3], [-1, 0, 0, 0], [0, S3 / 2, 0.5, 2]],
            40: [[-1, 0, 0, 0], [0, -0.5, S3 / 2, 2 * S3], [0, S3 / 2, 0.5, 2]]}
    for k, m in want.items():
        assert np.allclose(path[k], np.array(m), atol=1e-6), (k, path[k])
        assert np.isclose(np.linalg.norm(path[k][:, 3]), 4.0, atol=1e-5)
    assert np.array_equal(pose_spherical(0.0, -30.0, 4.0), path[40])


def make(monkeypatch, tmp_path, H=24, W=32, rays=100, test_images=20):
    from test_runner_cpu import make_runner
    r, fake = make_runner(monkeypatch, rays=rays, H=H, W=W, log_dir=str(tmp_path), exp_name="lego_t")
    render_cpu_backend.install(monkeypatch, fake)
    r.cfg.dataset.test.n_images, r.cfg.dataset.test.H, r.cfg.dataset.test.W = test_images, H, W
    return r, fake


def spy_render(monkeypatch):
    from jnerf_b200 import ops
    seen, real = [], ops.render_rays

    def spy(rays_o, rays_d, *a, **k):
        seen.append((rays_o.clone(), rays_d.clone(), a, k))
        return real(rays_o, rays_d, *a, **k)
    monkeypatch.setattr(ops, "render_rays", spy)
    return seen


def test_render_img_with_pose_uses_the_image_rays(monkeypatch, tmp_path):
    r, fake = make(monkeypatch, tmp_path)
    ds = r.dataset["train"]
    seen = spy_render(monkeypatch)
    for pose in (ds.poses[1], ds.poses[1][:3, :4]):                    # 4x4 and 3x4 poses
        img = r.render_img_with_pose(pose)
        assert img.shape == (ds.H, ds.W, 3) and torch.isfinite(img).all()
    o, d = ds.generate_rays_total_test(1)
    for so, sd, a, k in seen:
        assert torch.equal(so, o) and torch.equal(sd, d)               # the true W x H of a non-square frame, row-major
        assert a[11] == r.cfg.n_rays_per_batch and k["min_transmittance"] == 1e-4


def test_render_rays_leaves_the_rng_where_render_img_nosync_does(monkeypatch, tmp_path):
    r, fake = make(monkeypatch, tmp_path)
    s = r.sampler
    rng0 = s.rng.copy()
    img_ref, _ = r.render_img_nosync("train", 2)                        # 768 rays in 8 tiles of 100, the last one padded
    rng_ref = s.rng.copy()
    s.rng[:] = rng0
    o, d = r.dataset["train"].generate_rays_total_test(2)
    fake.calls.clear()
    rgb, alpha, n, rounds = r.render_rays(o, d, min_transmittance=0.0)
    assert fake.calls == ["render_rays"]
    assert np.array_equal(s.rng, rng_ref)
    assert np.array_equal(rng_ref, ol.pcg32_advance(rng0.copy(), 8 << 32))
    img = rgb + torch.tensor(r.background_color, dtype=torch.float32) * (1 - alpha)
    # numpy's exp in the stand-in's composite against the oracle's: a looser bar than the GPU test's 1e-5
    assert (img.reshape(img_ref.shape) - img_ref).abs().max() <= 1e-4
    assert n.sum() > 0 and rounds >= 1


def test_render_writes_an_mp4_of_the_camera_path(monkeypatch, tmp_path):
    cv2 = pytest.importorskip("cv2")
    r, fake = make(monkeypatch, tmp_path, H=16, W=24, rays=128)
    path = r.render()
    assert path == os.path.join(str(tmp_path), "lego_t", "demo.mp4")
    cap = cv2.VideoCapture(path)
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f)
    cap.release()
    assert len(frames) == 80 and all(f.shape == (16, 24, 3) for f in frames)
    assert fake.calls.count("render_rays") == 80
    with pytest.raises(ValueError, match="mp4"):
        r.render(save_path=str(tmp_path / "demo.avi"))
    # the file shows the true colours: a red frame decodes (OpenCV's BGR order) with its large value in the last channel
    red = torch.zeros((16, 24, 3))
    red[..., 0] = 1.0
    monkeypatch.setattr(r, "render_img_with_pose", lambda pose, min_transmittance=1e-4: red)
    r.render(save_path=str(tmp_path / "red.mp4"))
    ok, f = cv2.VideoCapture(str(tmp_path / "red.mp4")).read()
    assert ok and f[..., 2].mean() > 200 and f[..., 0].mean() < 60
    monkeypatch.setitem(sys.modules, "cv2", None)
    with pytest.raises(RuntimeError, match="OpenCV"):
        r.render(save_path=str(tmp_path / "x.mp4"))


def test_test_writes_the_views_and_matches_psnr(monkeypatch, tmp_path, capsys):
    from PIL import Image
    r, fake = make(monkeypatch, tmp_path)
    s = r.sampler
    rng0 = s.rng.copy()
    psnr = r.test(min_transmittance=0.0)
    assert "TOTAL TEST PSNR====" in capsys.readouterr().out
    ds = r.dataset["test"]
    assert ds is not None and ds.n_images == 2
    out = tmp_path / "lego_t" / "test"
    assert sorted(os.listdir(out)) == ["lego_t_gt_0.png", "lego_t_gt_1.png", "lego_t_r_0.png", "lego_t_r_1.png"]
    assert Image.open(out / "lego_t_r_0.png").mode == "RGB" and Image.open(out / "lego_t_r_0.png").size == (32, 24)
    s.rng[:] = rng0
    assert abs(psnr - r.psnr("test")) <= 0.01                          # same views, same jitter
    r.cfg.alpha_image = True
    r.render_test(save_path=str(tmp_path / "rgba"))
    assert Image.open(tmp_path / "rgba" / "lego_t_r_1.png").mode == "RGBA"
    assert Image.open(tmp_path / "rgba" / "lego_t_gt_1.png").mode == "RGB"


def test_a_test_split_without_images_saves_renders_only(monkeypatch, tmp_path, capsys):
    r, fake = make(monkeypatch, tmp_path)
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg
    r.dataset["test"] = build_from_cfg(r.cfg.dataset.test, DATASETS)
    r.dataset["test"].have_img = False                                 # runner.py:94, 173: no gt image, no PSNR
    r._render_ws = torch.zeros(4)
    assert r.test(min_transmittance=0.0) is None
    assert "TOTAL TEST PSNR" not in capsys.readouterr().out
    assert sorted(os.listdir(tmp_path / "lego_t" / "test")) == ["lego_t_r_0.png", "lego_t_r_1.png"]
    assert r._render_ws is None                                        # test() releases the renderer's workspace
    assert r.render_test(save_img=False) == []


def test_early_stop_bound_on_the_cpu_stand_in(monkeypatch, tmp_path):
    r, fake = make(monkeypatch, tmp_path)
    s = r.sampler
    o, d = r.dataset["train"].generate_rays_total_test(0)
    rng0 = s.rng.copy()
    rgb0, a0, n0, _ = r.render_rays(o, d, 0.0)
    eps = 0.05
    s.rng[:] = rng0
    rgb1, a1, n1, _ = r.render_rays(o, d, eps)
    assert (n1 <= n0).all()
    bg = torch.tensor([0.3, 0.6, 0.9])
    diff = (rgb1 + bg * (1 - a1)) - (rgb0 + bg * (1 - a0))
    assert diff.abs().max() <= eps * (1 + 0.9) + 1e-5


def test_c_abi_rejects_malformed_render_arguments():
    from jnerf_b200 import lib
    L = lib.load()
    lay = np.zeros(4, np.uint64)
    with pytest.raises(lib.NgpError, match="capacity"):
        lib.call("ngp_render_workspace_bytes", 10, 0, lay.ctypes.data)
    lib.call("ngp_render_workspace_bytes", 10, 64, lay.ctypes.data)
    assert lay[0] >= 10 * 28 + 64 * 40 and lay[1] < lay[2] < lay[0] and lay[3] < lay[0]
    fake_ws = 1 << 20                                                    # never dereferenced: the checks come first
    n = np.zeros(1, np.uint32)
    npp = n.ctypes.data_as(ctypes.c_void_p)

    def init(capacity, ws, tile):
        return lib.call("ngp_render_init", None, 10, capacity, ws, 0.0, 1.0, None, None, 0.004, 0.2, 5, 1, 1, 1, tile, None, None, None, npp)
    with pytest.raises(lib.NgpError, match="capacity"):
        init(0, fake_ws, 64)
    with pytest.raises(lib.NgpError, match="workspace"):
        init(64, None, 64)
    with pytest.raises(lib.NgpError, match="jitter_tile"):
        init(64, fake_ws, 0)

    def march(capacity, ws, n_alive, k):
        return lib.call("ngp_render_march_round", None, 10, capacity, ws, n_alive, k, 0.0, 1.0, None, None, None, 0.004, 5, 1)
    with pytest.raises(lib.NgpError, match="capacity"):
        march(0, fake_ws, 1, 1)
    with pytest.raises(lib.NgpError, match="workspace"):
        march(64, None, 1, 1)
    with pytest.raises(lib.NgpError, match="k_steps"):
        march(64, fake_ws, 1, 0)
    with pytest.raises(lib.NgpError, match="k_steps"):
        march(64, fake_ws, 1, 65)
    with pytest.raises(lib.NgpError, match="n_alive"):
        march(64, fake_ws, 11, 1)

    def composite(capacity, ws, n_alive, k):
        return lib.call("ngp_render_composite_round", None, 10, capacity, ws, n_alive, k, 1e-4, 5, None, None, None, npp)
    with pytest.raises(lib.NgpError, match="capacity"):
        composite(0, fake_ws, 1, 1)
    with pytest.raises(lib.NgpError, match="workspace"):
        composite(64, None, 1, 1)
    with pytest.raises(lib.NgpError, match="k_steps"):
        composite(64, fake_ws, 1, 0)
    with pytest.raises(lib.NgpError, match="n_alive"):
        composite(64, fake_ws, 11, 1)
    assert L.ngp_render_workspace_bytes is not None
