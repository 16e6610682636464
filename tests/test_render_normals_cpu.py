"""Normal maps without a GPU: the C-ABI argument checks of ngp_density_grad and of the normal composite, normal_from_sum (normalisation,
zeros and the model-to-NeRF axis rotation against matrix_nerf2ngp), the normal outputs of Runner.render_normal_with_pose / test / render
through a normals-capable stand-in of ops.render_rays, and a ptxas check that the density-gradient kernel does not spill."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import render_cpu_backend
from test_render_depth_cpu import install_depth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def install_normals(monkeypatch, fake):
    """test_render_depth_cpu's stand-in plus a `normals` argument.  Its normal sum is alpha * (o - 0.5) / |o - 0.5|: every covered pixel's
    normal points from the scene centre to its camera, so in NeRF world axes it is the unit camera position of the pose."""
    seen_depth = install_depth(monkeypatch, fake)
    import jnerf_b200.ops as real_ops
    inner = real_ops.render_rays
    seen = []

    def render_rays(rays_o, rays_d, *a, normals=False, **k):
        seen.append(normals)
        out = inner(rays_o, rays_d, *a, **k)
        if not normals:
            return out
        v = rays_o.float() - 0.5
        return out + (out[1] * v / v.norm(dim=1, keepdim=True),)
    monkeypatch.setattr(real_ops, "render_rays", render_rays)
    return seen, seen_depth


def make(monkeypatch, tmp_path, H=12, W=16, rays=64):
    from test_runner_cpu import make_runner
    r, fake = make_runner(monkeypatch, rays=rays, H=H, W=W, log_dir=str(tmp_path), exp_name="lego_t")
    seen, seen_depth = install_normals(monkeypatch, fake)
    r.cfg.dataset.test.n_images, r.cfg.dataset.test.H, r.cfg.dataset.test.W = 20, H, W
    return r, fake, seen, seen_depth


def test_normal_from_sum_normalises_zeroes_and_rotates():
    from jnerf_b200.plugin.dataset import matrix_nerf2ngp
    from jnerf_b200.runner import normal_from_sum
    rng = np.random.default_rng(0)
    nerf = rng.normal(size=(64, 3))
    nerf /= np.linalg.norm(nerf, axis=1, keepdims=True)
    # the linear part of the dataset's NeRF -> NGP map, whatever its scale, offset and camera-axis flips
    for scale, offset, cp in ((0.33, (0.5, 0.5, 0.5), (1, -1, -1)), (0.05, (0.2, 0.7, 0.5), (1, 1, 1))):
        P = matrix_nerf2ngp(np.eye(4, dtype=np.float32)[:3], 1.0, (0, 0, 0), (1, 1, 1))[:, :3].astype(np.float64)
        m = matrix_nerf2ngp(np.concatenate([np.eye(3), np.zeros((3, 1))], 1), scale, offset, cp)
        assert np.allclose(m[:, :3] @ np.diag(cp), P)                    # correct_pose flips camera axes; the world axes are P's
        ngp = nerf @ P.T                                                 # model-axes directions of the NeRF ones
        alpha = torch.rand(64, 1, dtype=torch.float32) * 0.9 + 0.1
        N = torch.from_numpy(ngp).float() * alpha * 0.37                 # any positive length
        n = normal_from_sum(N, alpha)
        assert n.shape == (64, 3) and n.dtype == torch.float32
        assert torch.allclose(n, torch.from_numpy(nerf).float(), atol=1e-6)
    N = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.3, 0.0], [2.0, 0.0, 0.0], [0.0, 0.0, -1e-30]])
    alpha = torch.tensor([[1.0], [0.0], [0.5], [1.0]])
    n = normal_from_sum(N, alpha)
    assert (n[0] == 0).all() and (n[1] == 0).all()                       # |N| 0 or alpha 0: no normal, not a division by zero
    assert torch.equal(n[2], torch.tensor([0.0, 1.0, 0.0]))              # model x is NeRF y
    assert torch.equal(n[3], torch.tensor([-1.0, 0.0, 0.0]))             # model z is NeRF x; a tiny sum still normalises
    assert normal_from_sum(torch.zeros(2, 4, 3), torch.ones(2, 4, 1)).shape == (2, 4, 3)


def test_normal_to_rgb_maps_minus_one_to_one():
    from jnerf_b200.runner import normal_to_rgb
    n = torch.tensor([[[1.0, 0.0, -1.0], [0.0, 0.0, 1.0]]])
    a = torch.tensor([[[1.0], [0.0]]])
    rgb = normal_to_rgb(n, a)
    assert rgb.dtype == np.uint8 and rgb.shape == (1, 2, 3)
    assert list(rgb[0, 0]) == [255, 128, 0] and list(rgb[0, 1]) == [0, 0, 0]


def test_render_normal_with_pose_points_in_nerf_axes(monkeypatch, tmp_path):
    r, fake, seen, _ = make(monkeypatch, tmp_path)
    ds = r.dataset["train"]
    img, normal, alpha = r.render_normal_with_pose(ds.poses[1])
    assert img.shape == (12, 16, 3) and normal.shape == (12, 16, 3) and alpha.shape == (12, 16, 1) and seen == [True]
    cam = np.asarray(ds.poses[1], np.float64)[:3, 3]
    want = torch.tensor(cam / np.linalg.norm(cam), dtype=torch.float32)
    a = alpha[..., 0]
    assert (a > 0).any() and (a == 0).any()
    assert torch.allclose(normal[a > 0], want.expand(int((a > 0).sum()), 3), atol=1e-5)
    assert (normal[a == 0] == 0).all()
    # the colour image is the one render_img_with_pose gives under the same jitter
    s = r.sampler
    s.rng[:] = rng0 = s.rng.copy()
    img1, _, _ = r.render_normal_with_pose(ds.poses[1])
    s.rng[:] = rng0
    assert torch.equal(img1, r.render_img_with_pose(ds.poses[1]))


def test_render_rays_returns_normals_last(monkeypatch, tmp_path):
    r, fake, seen, seen_depth = make(monkeypatch, tmp_path)
    o, d = r.dataset["train"].generate_rays_total_test(0)
    assert len(r.render_rays(o, d)) == 4 and seen == [False]
    out = r.render_rays(o, d, normals=True)
    assert len(out) == 5 and out[4].shape == (o.shape[0], 3) and seen == [False, True] and seen_depth[-1] is False
    out = r.render_rays(o, d, depth=True, normals=True)
    assert len(out) == 6 and out[4].shape == (o.shape[0],) and out[5].shape == (o.shape[0], 3) and seen_depth[-1] is True
    r.fast = False                                                       # a model without the fused network has no density gradient
    with pytest.raises(NotImplementedError, match="normal"):
        r.render_rays(o, d, normals=True)
    with pytest.raises(NotImplementedError, match="normal"):
        r.render(normals=True)


def test_ops_render_rays_refuses_normals_for_another_network():
    from jnerf_b200 import ops
    with pytest.raises(NotImplementedError, match="fused NGP"):
        ops.render_rays(torch.zeros(1, 3), torch.ones(1, 3), None, (0, 1), 0, 0, 5, False, np.zeros(2, np.uint64), None, None, None, None, 1,
                        net=lambda *a: None, normals=True)


def test_test_writes_normal_maps_from_the_same_render(monkeypatch, tmp_path):
    from PIL import Image
    r, fake, seen, seen_depth = make(monkeypatch, tmp_path)
    fake.calls.clear()
    r.test(min_transmittance=0.0, depth=True, normals=True)
    out = tmp_path / "lego_t" / "test"
    names = sorted(os.listdir(out))
    assert [f for f in names if "normal" in f] == ["lego_t_normal_0.npy", "lego_t_normal_0.png", "lego_t_normal_1.npy", "lego_t_normal_1.png"]
    assert len([f for f in names if "depth" in f]) == 4 and len(names) == 12
    assert fake.calls.count("render_rays") == 2 and seen == [True, True] and seen_depth == [True, True]   # one render per view
    ds = r.dataset["test"]
    for i in range(2):
        n = np.load(out / f"lego_t_normal_{i}.npy")
        png = np.asarray(Image.open(out / f"lego_t_normal_{i}.png"))
        assert n.dtype == np.float32 and n.shape == (12, 16, 3) and png.dtype == np.uint8 and png.shape == (12, 16, 3)
        covered = np.abs(n).sum(-1) > 0
        cam = np.asarray(ds.poses[i], np.float64)[:3, 3]
        assert covered.any() and np.allclose(n[covered], cam / np.linalg.norm(cam), atol=1e-5)
        assert np.allclose(np.linalg.norm(n[covered], axis=-1), 1, atol=1e-5)
        assert (png[~covered] == 0).all()
        alpha = np.load(out / f"lego_t_depth_{i}.npy") > 0                 # the depth and normal maps cover the same pixels
        assert (alpha == covered).all()
    seen.clear()
    r.render_test(save_path=str(tmp_path / "plain"))
    assert seen == [False, False] and not any("normal" in f for f in os.listdir(tmp_path / "plain"))


def test_render_writes_a_normal_video_beside_the_colour_one(monkeypatch, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from jnerf_b200.utils.camera_path import path_spherical
    r, fake, seen, _ = make(monkeypatch, tmp_path, H=16, W=24, rays=128)
    fake.calls.clear()
    path = r.render(normals=True, poses=path_spherical(6))
    npath = os.path.join(str(tmp_path), "lego_t", "demo_normal.mp4")

    def frames(p):
        cap, out = cv2.VideoCapture(p), []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            out.append(f)
        cap.release()
        return out
    col, nrm = frames(path), frames(npath)
    assert len(col) == len(nrm) == 6 and all(f.shape == (16, 24, 3) for f in col + nrm)
    assert fake.calls.count("render_rays") == 6 and seen == [True] * 6 and not os.path.exists(npath[:-11] + "_depth.mp4")


def test_c_abi_rejects_malformed_normal_arguments():
    from jnerf_b200 import lib
    lib.load()
    n = np.zeros(1, np.uint32)
    npp = n.ctypes.data_as(ctypes.c_void_p)
    fake = 1 << 20                                                        # never dereferenced: the checks come first

    def composite(capacity, ws, n_alive, k, grad=fake, normal=fake, depth=None):
        return lib.call("ngp_render_composite_round_normals", None, 10, capacity, ws, n_alive, k, 1e-4, 5, None, None, None, grad, normal, depth,
                        npp)
    with pytest.raises(lib.NgpError, match="grad_rows"):
        composite(64, fake, 1, 1, grad=None)
    with pytest.raises(lib.NgpError, match="normal_out"):
        composite(64, fake, 1, 1, normal=None)
    with pytest.raises(lib.NgpError, match="capacity"):
        composite(0, fake, 1, 1)
    with pytest.raises(lib.NgpError, match="workspace"):
        composite(64, None, 1, 1)
    with pytest.raises(lib.NgpError, match="k_steps"):
        composite(64, fake, 1, 0)
    with pytest.raises(lib.NgpError, match="n_alive"):
        composite(64, fake, 11, 1, depth=fake)
    assert composite(64, fake, 0, 1) == 0 and composite(64, fake, 0, 1, depth=fake) == 0 and n[0] == 0
    assert lib.KERNELS_PER_CALL["ngp_render_composite_round_normals"] == lib.KERNELS_PER_CALL["ngp_render_composite_round"]

    def grad(n_max, coords=fake, grid=fake, levels=fake, wd=fake, out=fake):
        return lib.call("ngp_density_grad", None, n_max, None, coords, grid, levels, wd, out)
    for k in ("coords", "grid", "levels", "wd"):
        with pytest.raises(lib.NgpError, match="coords, grid, levels and w_density are required"):
            grad(5, **{k: None})
    with pytest.raises(lib.NgpError, match="grad_out"):
        grad(5, out=None)
    assert grad(0, None, None, None, None, None) == 0                     # no rows: nothing to check or launch
    assert lib.KERNELS_PER_CALL["ngp_density_grad"] == 1


def test_density_grad_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc is not installed")
    from jnerf_b200 import build
    src = os.path.join(build.CSRC, "density_grad.cu")
    r = subprocess.run([nvcc] + build.ARCH + build.COMMON + build.SOURCES["density_grad.cu"] + ["-Xptxas", "-v", "-c", src, "-o",
                        str(tmp_path / "density_grad.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    blocks = re.findall(r"Compiling entry function '(\w+)'.*?Used (\d+) registers", log, flags=re.S)
    assert [name for name, _ in blocks if "density_grad_kernel" in name], log[-2000:]
    assert re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log) and \
        all(a == "0" and b == "0" for a, b in re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)), log[-2000:]
    for name, regs in blocks:
        if "density_grad_kernel" in name:
            assert int(regs) * 640 <= 65536, regs                        # the 640-thread CTA fits the register file
