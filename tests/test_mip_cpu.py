"""Mip-NeRF host logic without a GPU: mip_cfg against the reference's mip_base.py, the flat layout and its reference names (skip and view
column permutations), Blender on the reduced fox capture, the LinearLog sequence, the pcg32 offsets of the sampler kernels, the new
kernels compiling for sm_90a without spills, and MipRunner steps / test() / checkpoints / refusals with the operators swapped for the
torch restatement of tests/mip_cpu_backend.py."""
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def _reference_tree():
    if os.environ.get("NGP_REF"):
        return os.environ["NGP_REF"]
    m = re.search(r"^NGP_REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M)
    return m.group(1) if m else ""


def test_mip_cfg_is_mip_base_key_for_key():
    ref_cfg = os.path.join(_reference_tree(), "contrib", "mipnerf", "projects", "mipnerf", "configs", "mip_base.py")
    if not os.path.exists(ref_cfg):
        pytest.skip("reference tree not present")
    from jnerf_b200.mip_runner import mip_cfg
    ns = {}
    exec(open(ref_cfg).read(), ns)
    ref = {k: v for k, v in ns.items() if not k.startswith("__")}
    got = mip_cfg(synthetic=False)
    # the one documented difference: near / far also go into the dataset dicts, where Blender reads them
    for split in ("train", "val", "test"):
        assert (got["dataset"][split].pop("near"), got["dataset"][split].pop("far")) == (2.0, 6.0)
    assert got == ref


def test_flat_layout_and_reference_names():
    from jnerf_b200.plugin import mip, nerf
    g = torch.Generator().manual_seed(0)
    ref = {name: ((torch.rand((o, i), generator=g) - 0.5).half().float(), (torch.rand(o, generator=g) - 0.5).half().float())
           for name, ((o, i), _, _, _) in mip.REF_LAYERS.items()}
    flat = mip.pack(ref)
    assert flat.numel() == nerf.N_PARAMS
    back = mip.unpack(flat)
    for name, (W, b) in ref.items():
        assert torch.equal(back[name][0], W) and torch.equal(back[name][1], b)
    n_ref = sum(W.numel() + b.numel() for W, b in ref.values())
    assert int((flat != 0).sum()) <= n_ref
    # layers.5.0 reads [h4 (256), enc (48)]; the kernel reads [enc (64 padded), h4]
    W5 = flat[nerf.W_OFF[5]:nerf.W_OFF[5] + 256 * 320].view(256, 320).float()
    assert torch.equal(W5[:, :48], ref["layers.5.0"][0][:, 256:]) and torch.equal(W5[:, 64:], ref["layers.5.0"][0][:, :256])
    assert not W5[:, 48:64].any()
    # view_layers.0.0: reference column 256 + 3 + 3k + d (sin of degree k) is kernel column 256 + 3 + 6k + d, cosines 3 further
    W9 = flat[nerf.W_OFF[9]:nerf.W_OFF[9] + 128 * 288].view(128, 288).float()
    Wr = ref["view_layers.0.0"][0]
    for k in range(4):
        for d in range(3):
            assert torch.equal(W9[:, 259 + 6 * k + d], Wr[:, 259 + 3 * k + d])
            assert torch.equal(W9[:, 262 + 6 * k + d], Wr[:, 271 + 3 * k + d])
    assert torch.equal(W9[:, :259], Wr[:, :259]) and not W9[:, 283:].any()


def test_blender_on_the_reduced_fox_capture(tmp_path, monkeypatch):
    """Blender reads the capture's transforms json as nerf_datasets.py:73-150 does (frames without an image skipped, focal from fl_x), and
    its rays are the reference's numpy ray generation (radii from vertically adjacent pixels, the last row taking dx[-2] as :231 does)."""
    import mip_cpu_backend
    fake = mip_cpu_backend.install(monkeypatch)
    from make_fox_small import materialise
    from jnerf_b200.plugin import mip
    root = materialise(str(tmp_path / "fox"))
    import json
    for split in ("train", "test"):                                  # NeRF-synthetic's "./" prefix, which nerf_datasets.py:102 strips
        p = os.path.join(root, f"transforms_{split}.json")
        jd = json.load(open(p))
        for fr in jd["frames"]:
            fr["file_path"] = "./" + fr["file_path"]
        json.dump(jd, open(p, "w"))
    ds = mip.Blender(root, 64, mode="train", near=2.0, far=6.0)
    c = np.load(os.path.join(ROOT, "tests", "golden", "fox_small", "capture.npz"))
    assert ds.n_images == int(c["train_present"].sum()) == 50 and (ds.W, ds.H) == (180, 320)
    assert ds.focal == pytest.approx(float(c["intrinsics"][0]))
    mats = c["train_matrices"][c["train_present"]][:, :3, :4].astype(np.float32)
    assert np.array_equal(ds.c2w.numpy(), mats.reshape(-1, 12))
    rays, target = ds.image_rays(3)
    assert fake.calls.count("mip_rays") == 1 and rays.shape == (180 * 320, 12) and target.shape == (180 * 320, 3)
    # radii against an independent restatement: |d(y) - d(y+1)| of the direction image, * 2 / sqrt(12); the last row takes dx[-2]
    x, y = np.meshgrid(np.arange(180), np.arange(320), indexing="xy")
    f = float(c["intrinsics"][0])
    cam = np.stack([(x - 90 + 0.5) / f, -(y - 160 + 0.5) / f, -np.ones_like(x, dtype=np.float64)], -1)
    d = cam @ mats[3][:3, :3].astype(np.float64).T
    dx = np.linalg.norm(d[:-1] - d[1:], axis=-1)
    radii = np.concatenate([dx, dx[-2:-1]], 0) * 2 / np.sqrt(12)
    got = rays[:, 9].numpy().reshape(320, 180)
    assert np.allclose(got, radii, rtol=1e-4, atol=0) and np.array_equal(got[-1], got[-3])
    assert np.allclose(rays[:, 3:6].numpy().reshape(320, 180, 3), d, rtol=1e-5, atol=1e-6)
    assert bool((rays[:, 10] == 2.0).all() and (rays[:, 11] == 6.0).all())
    # test split: frames[::10] of transforms_test.json; no val json in the capture
    assert mip.Blender(root, 64, mode="test").n_images == 1
    with pytest.raises(FileNotFoundError):
        mip.Blender(root, 64, mode="val")


def test_linearlog_sequence():
    from jnerf_b200.plugin.optim import LinearLog

    class Nested:
        lr = 8e-3
    adam = Nested()
    sched = LinearLog(adam, end_lr=5e-6, max_steps=40001, lr_delay_steps=2500, lr_delay_mult=0.01)
    for step in (0, 1, 100, 2499, 2500, 2501, 20000, 40001, 50000):
        delay = 0.01 + 0.99 * math.sin(0.5 * math.pi * min(max(step / 2500, 0), 1))
        t = min(max(step / 40001, 0), 1)
        want = delay * math.exp(math.log(8e-3) * (1 - t) + math.log(5e-6) * t)
        assert sched.lr_at(step) == pytest.approx(want, rel=2e-6), step
    got = [sched.advance_lr() for _ in range(3)]
    assert got == [sched.lr_at(0), sched.lr_at(1), sched.lr_at(2)] and adam.lr == got[-1] and sched.steps == 3
    no_delay = LinearLog(Nested(), end_lr=5e-6, max_steps=10)
    assert no_delay.lr_at(0) == pytest.approx(Nested.lr, rel=1e-6) and no_delay.lr_at(10) == pytest.approx(5e-6, rel=1e-6)


def test_pcg32_offsets_match_the_library():
    """Draw j of ray g is draw g * (S + 1) + j of the stream: the host restatement against the library's own pcg32 (ngp_pcg32_advance)."""
    import mip_cpu_backend
    from jnerf_b200 import ops
    rng = ops.pcg32_seed(1337)
    u = mip_cpu_backend.pcg32_uniforms(rng, 5, 7)
    flat = mip_cpu_backend.pcg32_uniforms(rng, 1, 35)[0]
    assert np.array_equal(u.reshape(-1), flat)
    r2 = ops.pcg32_advance(rng.copy(), 3 * 7)
    assert np.array_equal(mip_cpu_backend.pcg32_uniforms(r2, 1, 7)[0], u[3])
    assert (u >= 0).all() and (u < 1).all() and len(np.unique(u)) == u.size


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
@pytest.mark.parametrize("src,n_entries,extra", [("mip_sampler.cu", 8, ["-fmad=false"]), ("mip_mlp.cu", 2, [])])
def test_kernels_compile_for_sm90a_without_spills(tmp_path, src, n_entries, extra):
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I",
                        os.path.join(ROOT, "include"), *extra, "-Xptxas", "-v", "-c", os.path.join(ROOT, "jnerf_b200", "csrc", src), "-o",
                        str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == n_entries and len(spills) >= n_entries, r.stderr[-3000:]          # + non-inlined device functions
    assert all(int(a) == 0 and int(b) == 0 for a, b in spills), r.stderr[-3000:]


def _make_runner(seed, tmp_path, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.mip_runner import MipRunner, mip_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**mip_cfg(seed=seed, num_samples=16, log_dir=str(tmp_path), **over))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=4 if split == "train" else 20, H=12, W=16, batch_size=8)
    return MipRunner()


def test_runner_steps_test_and_checkpoints(monkeypatch, tmp_path, capsys):
    """A few MipRunner steps of the fp32 model with the Mip-NeRF operators swapped for the torch restatement: both levels run, autograd
    reaches every layer, LinearLog sets Adam's rate; test() writes PNGs and a PSNR; the .pt round trip; the refusals."""
    import mip_cpu_backend
    fake = mip_cpu_backend.install(monkeypatch)
    r = _make_runner(1, tmp_path)
    m = r.model
    assert not m.using_fp16 and isinstance(m.layers[5][0], torch.nn.Linear) and m.layers[5][0].in_features == 304
    p0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    fake.calls.clear()
    losses = [float(r.train_step()) for _ in range(3)]
    assert all(np.isfinite(losses))
    per_step = ["mip_rays", "mip_sample", "mip_encode", "mip_composite_fwd", "mip_resample", "mip_encode", "mip_composite_loss_bwd"]
    assert [c for c in fake.calls if c.startswith("mip_")] == per_step * 3
    assert all(not torch.equal(p0[k], v) for k, v in m.state_dict().items()), "every parameter moves"
    adam = r.optimizer._nested_optimizer
    assert adam.n_step == 3 and r.optimizer.steps == 3 and adam.lr == pytest.approx(r.optimizer.lr_at(2))
    psnr = r.test()
    out = tmp_path / "lego_sss" / "test"
    assert np.isfinite(psnr) and sorted(os.listdir(out)) == ["lego_sss_gt_0.png", "lego_sss_gt_1.png", "lego_sss_r_0.png", "lego_sss_r_1.png"]
    assert "TOTAL TEST PSNR====" in capsys.readouterr().out
    path = str(tmp_path / "mip.pt")
    r.save_ckpt(path)
    r2 = _make_runner(2, tmp_path)
    r2.load_ckpt(path)
    assert all(torch.equal(v, m.state_dict()[k]) for k, v in r2.model.state_dict().items())
    assert r2.cfg.m_training_step == 3 and r2.optimizer.steps == 3 and np.array_equal(r2.sampler.rng, r.sampler.rng)
    assert torch.equal(r2.optimizer._nested_optimizer.state[0].m, adam.state[0].m)
    for fn in (lambda: r.save_ckpt(str(tmp_path / "x.pkl")), lambda: r.load_ckpt(str(tmp_path / "x.pkl")), r.render, r.extract_mesh):
        with pytest.raises(NotImplementedError):
            fn()


def test_refusals_and_the_near_far_warning(monkeypatch, tmp_path, capsys):
    import mip_cpu_backend
    mip_cpu_backend.install(monkeypatch)
    from jnerf_b200.mip_runner import MipRunner
    with pytest.raises(NotImplementedError, match="density_noise"):
        _make_runner(1, tmp_path, density_noise=1.0)
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg
    with pytest.raises(NotImplementedError, match="Blenders"):
        build_from_cfg(dict(type="Blenders", root_dir="x", batch_size=8), DATASETS)
    with pytest.raises(NotImplementedError, match="data-parallel"):
        MipRunner(world_size=2)
    # mip_base.py as shipped: near / far only at the top level -> one warning naming them, and Blender keeps its [0, 1] defaults
    from jnerf_b200.mip_runner import mip_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    c = mip_cfg(num_samples=16, log_dir=str(tmp_path))
    for split in ("train", "val", "test"):
        del c["dataset"][split]["near"], c["dataset"][split]["far"]
    get_cfg().clear()
    update_cfg(**c)
    for split in ("train", "val", "test"):
        get_cfg().dataset[split].update(n_images=2, H=12, W=16, batch_size=8)
    capsys.readouterr()
    r = MipRunner()
    assert capsys.readouterr().out.count("WARNING: config keys near, far are not read") == 1
    assert (r.dataset["train"].near, r.dataset["train"].far) == (0.0, 1.0)
