"""pixelNeRF host logic without a GPU: rays, the fixture loader, the encoding's columns, the flat layout, the checkpoint, the projection's
mirror, the kernels' register / spill report, the encoder's weight check, and PixelNeRFRunner's train / test / video / checkpoint logic on
the float64 stand-in of its operators (tests/pixelnerf_cpu_backend.py)."""
import os
import re
import subprocess

import numpy as np
import torch

from jnerf_b200.plugin import pixelnerf as pn

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "pixelnerf_tiny.npz")


def test_rays_match_dataset_py():
    d = np.load(FIXTURE)
    H, W, f, c2w = 100, 100, float(d["focal"]), d["poses"][1]
    o, dd = pn.sample_rays_np(H, W, f, c2w)
    j, i = np.mgrid[0:H, 0:W].astype(np.float32)
    cam = np.stack([(i - W * .5 + 0.5) / f, -(j - H * .5 + 0.5) / f, -np.ones_like(i)], -1)
    assert np.allclose(dd, cam @ c2w[:3, :3].T, atol=1e-6) and np.array_equal(o[5, 7], c2w[:3, 3])


def test_fixture_loader_gives_14_batches_an_epoch():
    data = pn.TinyNerfData(FIXTURE, 3, device="cpu")
    assert data.rays.shape == (30000, 9) and data.images.shape == (8, 100, 100, 3)
    assert np.array_equal(data.rays[:10000, 6:9].numpy(), data.images[0].reshape(-1, 3))
    batches = list(data.batches(2048, torch.Generator().manual_seed(0)))
    assert len(batches) == 14 and all(b.shape == (2048, 9) for b in batches)
    assert len(torch.unique(torch.cat(batches)[:, :6], dim=0)) == 14 * 2048           # no ray twice in an epoch


def test_positional_encoding_columns():
    x, d = torch.tensor([[0.3, -1.2, 2.0]], dtype=torch.float64), torch.tensor([[0.0, 3.0, 4.0]], dtype=torch.float64)
    e = pn.positional_encoding(x, d)
    assert e.shape == (1, 42)
    assert torch.equal(e[0, :3], x[0])
    for i in range(6):
        assert torch.allclose(e[0, 3 + 6 * i:6 + 6 * i], torch.sin(2.0 ** i * x[0] * 1.5))
        assert torch.allclose(e[0, 6 + 6 * i:9 + 6 * i], torch.cos(2.0 ** i * x[0] * 1.5))
    assert torch.allclose(e[0, 39:], torch.tensor([0.0, 0.6, 0.8], dtype=torch.float64))


def test_flat_layout_round_trip_and_reference_names():
    s = pn.init_state(2)
    assert sum(v.numel() for v in s.values()) == pn.N_PARAMS == 3438596
    names = {k.rsplit(".", 1)[0] for k in s}
    assert names == {"mlp.0", "final_layer"} | {f"f1.{i}.{n}" for i in range(3) for n in ("img_mlp.0", "mlp.0", "mlp.2")} | \
        {f"f2.{i}.{n}" for i in range(2) for n in ("mlp.0", "mlp.2")}
    flat = pn.pack(s)
    assert flat.numel() == pn.N_FLAT
    w0, b0 = pn.flat_offsets()["mlp.0"]
    assert torch.all(flat[w0:b0].view(512, 64)[:, 42:] == 0)
    back = pn.unpack(flat)
    assert all(torch.equal(back[k], s[k]) for k in s)


def test_checkpoint_round_trip(tmp_path):
    m = pn.PixelNeRF(seed=3, device="cpu")
    p = tmp_path / "net.pth"
    torch.save(m.reference_state(), p)
    m2 = pn.PixelNeRF(seed=4, device="cpu")
    m2.load_reference_state(torch.load(p, weights_only=True))
    assert torch.equal(m.master, m2.master) and torch.equal(m.params, m2.params)


def test_projection_mirror_and_pixel_aligned():
    """The pixel-centre rays of reference 0 land at (H-1-r, W-1-c) of its image frame with the reference's projection, at (r, c) with
    pixel_aligned (grid_sample's align_corners frame, scaled to the full-resolution image)."""
    d = np.load(FIXTURE)
    H, f, c2w = 100, float(d["focal"]), d["poses"][:3]
    cams = pn.pack_cams(c2w).double()
    o, dd = pn.sample_rays_np(H, H, f, c2w[0])
    pts = torch.from_numpy(o + 4.0 * dd).double().reshape(-1, 3)
    rc = np.stack(np.mgrid[0:H, 0:H], -1).reshape(-1, 2)[:, ::-1].astype(np.float64)     # (col, row)
    for aligned, want in ((False, (H - 1) - rc), (True, rc)):
        uv = pn.project(pts, cams, (H / 2) / f, aligned)[0].numpy()
        pix = (uv + 1) / 2 * (H - 1)
        assert np.abs(pix - want).max() < 0.51 + 1e-3, (aligned, np.abs(pix - want).max())


def test_ptxas_reports_no_spills():
    src = os.path.join(HERE, "..", "jnerf_b200", "csrc", "pixelnerf.cu")
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I",
                        os.path.join(HERE, "..", "include"), "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills)
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", r.stderr)]
    assert max(regs) <= 128                                   # two 256-thread CTAs an SM for the GEMM


# ---- PixelNeRFRunner's host logic on the float64 CPU stand-in of its operators ----------------------------------------------------------
def _tiny_capture(tmp_path, size=10):
    """The fixture's views reduced to size x size (block means), focal scaled with them."""
    d = np.load(FIXTURE)
    k = d["images"].shape[1] // size
    imgs = d["images"].reshape(-1, size, k, size, k, 3).mean((2, 4)).astype(np.float32)
    p = tmp_path / "tiny.npz"
    np.savez(p, images=imgs, poses=d["poses"], focal=d["focal"] / k)
    return str(p)


def _runner(monkeypatch, tmp_path, **over):
    import torchvision  # noqa: F401  (imported before the stand-in replaces torch.Generator, which torchvision's import annotates with)
    import pixelnerf_cpu_backend
    from jnerf_b200.pixelnerf_runner import PixelNeRFRunner, pixelnerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    fake = pixelnerf_cpu_backend.install(monkeypatch)
    get_cfg().clear()
    update_cfg(**pixelnerf_cfg(_tiny_capture(tmp_path), **dict(dict(batch_size=32, N_samples=(4, None), log_dir=str(tmp_path / "logs")), **over)))
    return PixelNeRFRunner(), fake


def test_runner_trains_tests_renders_and_checkpoints_on_the_cpu_stand_in(monkeypatch, tmp_path):
    import warnings
    warnings.simplefilter("ignore")
    r, fake = _runner(monkeypatch, tmp_path)
    assert r.data.rays.shape == (3 * 100, 9)
    p0 = r.model.master.clone()
    losses = []
    for batch in r.data.batches(32, r.gen):
        losses.append(float(r.train_step(batch)))
    assert len(losses) == 9 and all(np.isfinite(losses)) and r.step == 9
    assert not torch.equal(r.model.master, p0) and torch.equal(r.model.params, r.model.master.half())
    w0, b0 = pn.flat_offsets()["mlp.0"]
    assert torch.all(r.model.master[w0:b0].view(512, 64)[:, 42:] == 0)     # the pad columns never move
    assert fake.calls.count("pixelnerf_bwd") == 9 and fake.calls.count("adam_ema") == 9
    # test: one PNG pair per held-out view, a finite mean PSNR
    psnr = r.test(save_dir=str(tmp_path / "test"))
    assert np.isfinite(psnr) and sorted(os.listdir(tmp_path / "test")) == sorted([f"r_{i}.png" for i in range(3, 8)] + [f"gt_{i}.png" for i in range(3, 8)])
    assert r.render_img_with_pose(r.data.poses[4]).shape == (10, 10, 3)
    # video: the 120 frames of test_utils.py
    import cv2
    path = r.render(str(tmp_path / "v.mp4"))
    cap = cv2.VideoCapture(path)
    n = 0
    while cap.read()[0]:
        n += 1
    assert n == 120
    # checkpoint: a .pth of fp32 tensors under the reference's names, read back by a fresh runner
    r.save_ckpt(str(tmp_path / "net.pth"))
    sd = torch.load(tmp_path / "net.pth", weights_only=True)
    assert set(sd) == {f"{n}.{w}" for n, *_ in pn.LINEARS for w in ("weight", "bias")} and all(v.dtype == torch.float32 for v in sd.values())
    r2, _ = _runner(monkeypatch, tmp_path, seed=5)
    assert not torch.equal(r2.model.master, r.model.master)
    r2.load_ckpt(str(tmp_path / "net.pth"))
    assert torch.equal(r2.model.master, r.model.master) and torch.equal(r2.model.params, r.model.params)
    import pytest
    with pytest.raises(NotImplementedError):
        r.save_ckpt(str(tmp_path / "net.pkl"))
    with pytest.raises(NotImplementedError):
        r.extract_mesh()


def test_runner_refuses_what_it_does_not_support(monkeypatch, tmp_path):
    import pytest
    from jnerf_b200.pixelnerf_runner import PixelNeRFRunner
    for over in (dict(noise_std=0.1), dict(N_samples=(64, 128))):
        with pytest.raises(NotImplementedError):
            _runner(monkeypatch, tmp_path, **over)
    _runner(monkeypatch, tmp_path)
    with pytest.raises(NotImplementedError):
        PixelNeRFRunner(world_size=2)


def test_encoder_weights_must_be_a_resnet34_state_dict():
    import pytest
    import torchvision
    sd = torchvision.models.resnet34(weights=None).state_dict()
    pn.ImageEncoder({k: v for k, v in sd.items() if not k.startswith("fc.")})
    with pytest.raises(ValueError):
        pn.ImageEncoder({f"module.{k}": v for k, v in sd.items()})
    torch.manual_seed(123)
    a = torch.rand(3)
    torch.manual_seed(123)
    pn.ImageEncoder(seed=0)
    assert torch.equal(torch.rand(3), a)                     # the encoder's seed leaves the caller's RNG alone
