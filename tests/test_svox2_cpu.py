"""Plenoxels host logic without a GPU: svox2_cfg against the reference's svox2_base.py, SvoxNeRFDataset on a Blender-layout fixture, the
learning-rate schedule, the npz checkpoint (ours and one laid out as the reference writes it), TV cell selection, the kernels compiling
for sm_90a without spills, and Svox2Runner steps / resample / eval / test / checkpoints / refusals with the operators swapped for the
restatement of tests/svox_cpu_backend.py."""
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _reference_tree():
    if os.environ.get("NGP_REF"):
        return os.environ["NGP_REF"]
    m = re.search(r"^NGP_REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M)
    return m.group(1) if m else ""


def test_svox2_cfg_is_svox2_base_key_for_key():
    path = os.path.join(_reference_tree(), "contrib", "plenoxel", "projects", "svox2", "configs", "svox2_base.py")
    if not os.path.exists(path):
        pytest.skip("reference tree not present")
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.svox2_runner import svox2_cfg
    from jnerf_b200.utils.config import init_cfg
    from jnerf_b200.utils.registry import DATASETS, LOSSES, NETWORKS
    ns = {}
    exec(open(path).read(), ns)
    assert svox2_cfg() == {k: v for k, v in ns.items() if not k.startswith("__")}
    cfg = init_cfg(path)                                   # the shipped file, unchanged
    assert NETWORKS.get(cfg.model.type) and DATASETS.get(cfg.dataset.train.type) and LOSSES.get(cfg.loss.type)


def _write_blender(root, n=3, H=8, W=8, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    from jnerf_b200.plugin.dataset import synthetic_cameras
    os.makedirs(os.path.join(root, "train"), exist_ok=True)
    frames, imgs = [], []
    for i, m in enumerate(synthetic_cameras(n, radius=2.5, seed=seed)):
        im = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
        Image.fromarray(im).save(os.path.join(root, "train", f"r_{i}.png"))
        frames.append({"file_path": f"./train/r_{i}", "transform_matrix": np.asarray(m).tolist()})
        imgs.append(im)
    for split in ("train", "test"):
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": 0.69, "frames": frames}, f)
    os.makedirs(os.path.join(root, "test"), exist_ok=True)
    for i in range(n):
        Image.fromarray(imgs[i]).save(os.path.join(root, "test", f"r_{i}.png"))
    return frames, imgs


def test_dataset_on_a_blender_fixture(tmp_path, monkeypatch):
    import svox_cpu_backend
    svox_cpu_backend.install(monkeypatch)
    from jnerf_b200.plugin.svox2 import SvoxNeRFDataset
    frames, imgs = _write_blender(str(tmp_path))
    ds = SvoxNeRFDataset(str(tmp_path), "train", epoch_size=100)
    m = np.array(frames[1]["transform_matrix"], np.float32) @ np.diag([1, -1, -1, 1]).astype(np.float32)
    m[:3, 3] *= np.float32(2 / 3)
    np.testing.assert_allclose(ds.c2w[1].numpy(), m, rtol=1e-6, atol=1e-7)
    assert ds.focal == pytest.approx(0.5 * 8 / math.tan(0.5 * 0.69))
    assert ds.intrins["cx"] == 4.0 and ds.n_rays == 3 * 64
    im = imgs[2].astype(np.float32) / 255.0
    np.testing.assert_allclose(ds.gt_image(2).numpy(), im[..., :3] * im[..., 3:] + (1 - im[..., 3:]), rtol=1e-6, atol=1e-6)


def test_lr_schedule_against_the_reference_formula():
    from jnerf_b200.svox2_runner import get_expon_lr_func

    def ref(step, lr0, lr1, delay, mult, max_steps):
        rate = mult + (1 - mult) * math.sin(0.5 * math.pi * min(max(step / delay, 0), 1)) if delay > 0 else 1.0
        t = min(max(step / max_steps, 0), 1)
        return rate * math.exp(math.log(lr0) * (1 - t) + math.log(lr1) * t)
    f = get_expon_lr_func(30.0, 0.05, 15000, 0.01, 250000)
    for s in (0, 14999, 15000, 15001, 125000, 250000, 300000):
        assert f(s) == pytest.approx(ref(s, 30.0, 0.05, 15000, 0.01, 250000), rel=1e-12)
    assert f(0) == pytest.approx(0.3) and f(250000) == pytest.approx(0.05)
    g = get_expon_lr_func(0.01, 5e-6, 0, 0.01, 250000)
    assert g(0) == pytest.approx(0.01) and g(125000) == pytest.approx(math.sqrt(0.01 * 5e-6)) and g(-1) == 0.0


def test_tv_cells_wrap_around():
    import svox_cpu_backend as ref
    from jnerf_b200.svox2_runner import tv_cells
    gen = torch.Generator().manual_seed(3)
    starts = [tv_cells(1000, 0.01, gen) for _ in range(200)]
    assert all(n == 10 and 0 <= s < 1000 for s, n in starts)
    assert tv_cells(10, 0.01, gen)[1] == 1                          # max(int(0.01 * G), 1)
    # the cells are start .. start + n - 1 mod G: the last ones of a start near the end are the grid's first cells
    links = np.arange(4 * 4 * 4, dtype=np.int32).reshape(4, 4, 4)
    data = np.random.default_rng(0).random((64, 1)).astype(np.float32)
    g_wrap = ref.tv_grad(links, data, 60, 8, 1.0, False)
    g_split = ref.tv_grad(links, data, 60, 4, 1.0, False) + ref.tv_grad(links, data, 0, 4, 1.0, False)
    np.testing.assert_allclose(g_wrap, g_split, rtol=0, atol=1e-15)


def test_npz_round_trip_and_the_reference_layout(tmp_path, monkeypatch):
    import svox_cpu_backend
    svox_cpu_backend.install(monkeypatch)
    from jnerf_b200.plugin.svox2 import SparseGrid
    g = SparseGrid(8, radius=[1.0, 1.5, 2.0], center=[0.1, 0.0, -0.2], use_z_order=True, use_sphere_bound=True)
    g.density_data.copy_(torch.rand(g.capacity, 1))
    g.sh_data.copy_(torch.randn(g.capacity, 27))
    g.save(str(tmp_path / "a.npz"))
    z = np.load(tmp_path / "a.npz")
    assert set(z.files) == {"radius", "center", "links", "density_data", "sh_data", "basis_type"}
    assert z["sh_data"].dtype == np.float16 and z["density_data"].dtype == np.float32 and z["links"].dtype == np.int32
    h = SparseGrid.load(str(tmp_path / "a.npz"))
    assert torch.equal(h._links, g._links) and torch.equal(h.density_data, g.density_data) and h.capacity == g.capacity
    assert torch.equal(h.sh_data, g.sh_data.half().float())
    np.testing.assert_array_equal(h._offset.numpy(), g._offset.numpy())
    # a file as the reference's np.savez writes it: radius / center float32 (3,), links int32 (X, Y, Z), basis_type a 0-d int
    links = np.full((4, 4, 4), -1, np.int32)
    links[1:3, 1:3, 1:3] = np.arange(8, dtype=np.int32).reshape(2, 2, 2)
    np.savez(tmp_path / "ref.npz", radius=np.array([1, 1, 1], np.float32), center=np.zeros(3, np.float32), links=links,
             density_data=np.arange(8, dtype=np.float32).reshape(8, 1), sh_data=np.ones((8, 27), np.float16), basis_type=np.array(1))
    r = SparseGrid.load(str(tmp_path / "ref.npz"))
    assert r.capacity == 8 and r._links.shape == (4, 4, 4) and r.sh_data.dtype == torch.float32 and float(r.density_data[7]) == 7.0


def test_sphere_bound_links_are_morton_ranks(monkeypatch):
    import svox_cpu_backend
    svox_cpu_backend.install(monkeypatch)
    from jnerf_b200.plugin.svox2 import SparseGrid, gen_morton
    g = SparseGrid(8, use_z_order=True, use_sphere_bound=True)
    lk = g._links.numpy().reshape(-1)
    kept = lk >= 0
    assert g.capacity == kept.sum() < 512 and lk[kept].max() == g.capacity - 1
    mort = gen_morton(8).reshape(-1)[kept]
    assert np.array_equal(np.argsort(np.argsort(mort)), lk[kept])     # the kept cells numbered in Morton order


@pytest.mark.parametrize("src", ["svox.cu"])
def test_kernels_compile_for_sm90a_without_spills(tmp_path, src):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I",
                        os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", os.path.join(ROOT, "jnerf_b200", "csrc", src), "-o",
                        str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    stack = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(stack) >= 9 and all(s == ("0", "0", "0") for s in stack), stack


def _runner(tmp_path, monkeypatch, **over):
    import svox_cpu_backend
    fake = svox_cpu_backend.install(monkeypatch)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.svox2_runner import Svox2Runner, svox2_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    _write_blender(str(tmp_path / "data"))
    get_cfg().clear()
    c = svox2_cfg(reso_list=[[8] * 3, [16] * 3], batch_size=16, epoch_size=2, upsamp_every=4, n_iters=6, log_dir=str(tmp_path / "logs"))
    for s in ("train", "test"):
        c["dataset"][s].update(root=str(tmp_path / "data"), epoch_size=2 * 16)
    c.update(over)
    update_cfg(**c)
    return Svox2Runner(), fake


def test_runner_steps_resample_eval_test_and_ckpt(monkeypatch, tmp_path, capsys):
    r, fake = _runner(tmp_path, monkeypatch)
    r.model.param_init(r.cfg)
    d0 = r.model.density_data.clone()
    se = r.train_step(0)
    assert se.shape == (16,) and torch.isfinite(se).all()
    assert not torch.equal(d0, r.model.density_data)
    assert int(r.optimizer.grad_density.abs().sum()) == 0               # the sweep cleared what it read
    r.train()
    assert r.model._links.shape == (16, 16, 16) and r.model.capacity == r.model.density_data.shape[0] == r.model.sh_data.shape[0]
    assert r.cfg.lambda_tv == 0.0 and r.cfg.lambda_tv_sh == 0.0          # tv_early_only after the upsample
    assert os.path.exists(r.ckpt_path) and os.path.isdir(os.path.join(r.save_path, "000000006"))
    assert "eval stats" in capsys.readouterr().out
    names = [c[0] if isinstance(c, tuple) else c for c in fake.calls]
    for op in ("svox_train_step", "svox_tv_grad", "svox_rmsprop", "svox_weight_render", "svox_dilate", "svox_compact", "svox_sample", "svox_render"):
        assert op in names, op
    psnr = r.test()
    assert math.isfinite(psnr) and "TOTAL TEST PSNR" in capsys.readouterr().out
    assert os.path.exists(os.path.join(r.save_path, "test", "lego_r_0.png"))
    img = r.render_img("test", 0)[0]
    r.save_ckpt(str(tmp_path / "c.npz"))
    r.load_ckpt(str(tmp_path / "c.npz"))
    assert r.model._links.shape == (16, 16, 16)
    assert torch.allclose(r.render_img("test", 0)[0], img, atol=2e-2)


def test_refusals(monkeypatch, tmp_path):
    from jnerf_b200.plugin.svox2 import SparseGrid
    with pytest.raises(NotImplementedError):
        SparseGrid(8, basis_type=4, device="cpu")
    with pytest.raises(NotImplementedError):
        SparseGrid(8, background_nlayers=2, device="cpu")
    for over in (dict(use_spheric_clip=True), dict(enable_random=True, random_sigma_std=1.0), dict(tv_logalpha=True), dict(weight_decay_sh=0.9)):
        with pytest.raises(NotImplementedError):
            _runner(tmp_path, monkeypatch, **over)
    r, _ = _runner(tmp_path, monkeypatch)
    with pytest.raises(NotImplementedError):
        r.render()
    with pytest.raises(NotImplementedError):
        r.extract_mesh()
