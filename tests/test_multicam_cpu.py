"""multicam.py's Mip-NeRF without a GPU: multicam_cfg against the reference's config, Blenders / Multicam on the written multiscale
stand-in (split selection, the ragged table, white compositing, factor 2, refusals), the rays of both datasets against the Blender
restatement, the 16-degree layer shapes, the new kernels compiling for sm_90a without spills, and MipRunner steps with the loss mask,
with the operators swapped for the restatements of tests/mip_cpu_backend.py and tests/multicam_cpu_backend.py."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 24, 32                             # levels 24x32, 12x16, 6x8, 3x4


def _reference_tree():
    if os.environ.get("NGP_REF"):
        return os.environ["NGP_REF"]
    m = re.search(r"^NGP_REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M)
    return m.group(1) if m else ""


def test_multicam_cfg_is_multicam_py_key_for_key():
    ref_cfg = os.path.join(_reference_tree(), "contrib", "mipnerf", "projects", "mipnerf", "configs", "multicam.py")
    if not os.path.exists(ref_cfg):
        pytest.skip("reference tree not present")
    from jnerf_b200.mip_runner import multicam_cfg
    ns = {}
    exec(open(ref_cfg).read(), ns)
    ref = {k: v for k, v in ns.items() if not k.startswith("__")}
    assert multicam_cfg(synthetic=False) == ref
    c = multicam_cfg(root_dir="/data/lego")
    assert c["dataset"]["test"]["data_dir"] == "/data/lego" and c["dataset_type"] == "Blenders"
    assert multicam_cfg()["dataset"]["train"]["type"] == "SyntheticMulticam"


@pytest.fixture
def stand_in(tmp_path, monkeypatch):
    import multicam_cpu_backend
    fake = multicam_cpu_backend.install(monkeypatch)
    from jnerf_b200.plugin import dataset as D
    root = str(tmp_path / "lego")
    D.write_synthetic_multicam(root, n_images=8, H=H, W=W, seed=2)
    return root, fake


def test_blenders_and_multicam_on_the_written_stand_in(stand_in):
    from PIL import Image
    from jnerf_b200.plugin import mip
    root, fake = stand_in
    meta = json.load(open(os.path.join(root, "metadata.json")))
    assert set(meta) == {"train", "val", "test"} and len(meta["train"]["file_path"]) == 8 * 4
    assert meta["train"]["lossmult"][:4] == [1.0, 4.0, 16.0, 64.0] and meta["train"]["width"][:4] == [32, 16, 8, 4]
    # pix2cam of level l: diag(1, -1, -1) K_l^-1, focal and principal point scaled by 2^-l
    p2c = np.array(meta["train"]["pix2cam"][1])
    assert p2c[0, 1] == 0 and p2c[1, 1] < 0 and p2c[2, 2] == -1 and p2c[0, 2] == pytest.approx(-8 * p2c[0, 0])

    mc = mip.Multicam(root, "train", batch_size=16)
    sizes = [(h, w) for w, h in zip(meta["train"]["width"], meta["train"]["height"])]
    assert mc.n_images == 32 and list(zip(mc.Hs, mc.Ws)) == sizes
    assert mc.offsets == [0] + np.cumsum([h * w for h, w in sizes]).tolist()
    img5 = np.asarray(Image.open(os.path.join(root, meta["train"]["file_path"][5])))
    assert np.array_equal(mc.table["images"][mc.offsets[5]:mc.offsets[6]].numpy(), img5.reshape(-1, 4))
    assert np.array_equal(mc.table["cams"][5].numpy(), mip.cam_row(meta["train"]["pix2cam"][5], meta["train"]["cam2world"][5], 4.0, 2.0, 6.0))
    rays, target, lossmult = next(mc)
    assert rays.shape == (16, 12) and target.shape == (16, 3) and fake.calls.count("mip_rays_multi") == 1
    # white compositing: the uint8 / 255 RGBA of the pixel, rgb a + (1 - a) in fp32
    r, t, _ = mc.rays_for(torch.arange(mc.offsets[5], mc.offsets[6], dtype=torch.int32))
    f = img5.reshape(-1, 4).astype(np.float32) / np.float32(255)
    assert np.array_equal(t.numpy(), f[:, :3] * f[:, 3:] + (np.float32(1) - f[:, 3:]))
    assert bool((r[:, 10] == 2).all() and (r[:, 11] == 6).all())
    # val / test: the first 20 entries of every key
    m = json.load(open(os.path.join(root, "metadata.json")))
    m["test"] = {k: v * 6 for k, v in m["test"].items()}                # 4 entries (one view, four levels) -> 24
    json.dump(m, open(os.path.join(root, "metadata.json"), "w"))
    ts = mip.Multicam(root, "test", batch_type="single_image", batch_size=4)
    assert ts.n_images == 20 and ts.Ws[:5] == [32, 16, 8, 4, 32]
    rays, target, lossmult = next(ts)
    assert len({int(x) for x in (rays[:, 9] > 0)}) == 1 and lossmult.unique().numel() == 1      # one image a batch
    with pytest.raises(ValueError, match="single_image"):
        mip.Multicam(root, "test")

    bl = mip.Blenders(root, "train", batch_size=16)
    assert bl.n_images == 8 and set(bl.Hs) == {H} and bl.focal == pytest.approx(0.5 * W / np.tan(0.5 * 0.6911112070083618))
    assert bool((next(bl)[2] == 1).all())
    assert np.array_equal(bl.table["images"][:H * W].numpy(), np.asarray(Image.open(os.path.join(root, "train", "r_0.png"))).reshape(-1, 4))
    tj = json.load(open(os.path.join(root, "transforms_test.json")))
    tj["frames"] = tj["frames"] * 25
    json.dump(tj, open(os.path.join(root, "transforms_test.json"), "w"))
    assert mip.Blenders(root, "test", batch_type="single_image").n_images == 20
    # factor 2: the 2x2 area mean of uint8 / 255 in fp32, stored as fp32 RGBA
    b2 = mip.Blenders(root, "train", factor=2)
    im0 = np.asarray(Image.open(os.path.join(root, "train", "r_0.png"))).astype(np.float32) / np.float32(255)
    want = ((im0[0::2, 0::2] + im0[0::2, 1::2]) + (im0[1::2, 0::2] + im0[1::2, 1::2])) * np.float32(0.25)
    assert b2.table["images"].dtype == torch.float32 and (b2.H, b2.W) == (H // 2, W // 2)
    assert np.array_equal(b2.table["images"][:H * W // 4].numpy(), want.reshape(-1, 4))
    with pytest.raises(ValueError, match="factor"):
        mip.Blenders(root, "train", factor=4)
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg
    with pytest.raises(NotImplementedError, match="Blenders.*data_dir"):
        build_from_cfg(dict(type="Blenders", root_dir="x", batch_size=8), DATASETS)
    with pytest.raises(NotImplementedError, match="Multicam.*mode"):
        mip.Multicam(root, "train", mode="train")


def test_rays_of_both_datasets_against_the_blender_restatement(stand_in):
    """Blenders' rays are Blender's (mip_cpu_backend.blender_rays_numpy); Multicam's, through the stand-in's pix2cam, are those of a Blender
    camera with the level's focal length; radii use the last-row rule (row H - 1 takes row H - 3's)."""
    import mip_cpu_backend
    from jnerf_b200.plugin import mip
    root, _ = stand_in
    bl = mip.Blenders(root, "train", white_bkgd=False)
    mc = mip.Multicam(root, "train", white_bkgd=False)
    for k in (0, 3):
        want = mip_cpu_backend.blender_rays_numpy(bl.table["cams"][k, 9:21].numpy(), bl.focal, W, H, 2.0, 6.0)
        got, tgt = bl.image_rays(k)
        assert np.allclose(got.numpy(), want, rtol=1e-5, atol=1e-6)
        for lvl in range(4):
            i = 4 * k + lvl
            h, w = mc.image_hw(i)
            want = mip_cpu_backend.blender_rays_numpy(mc.table["cams"][i, 9:21].numpy(), bl.focal / 2 ** lvl, w, h, 2.0, 6.0)
            got, _ = mc.image_rays(i)
            assert np.allclose(got.numpy(), want, rtol=1e-4, atol=1e-6), (k, lvl)
            rad = got[:, 9].numpy().reshape(h, w)
            assert np.array_equal(rad[-1], rad[-3])
            assert bool((mc.rays_for(torch.arange(mc.offsets[i], mc.offsets[i + 1], dtype=torch.int32))[2] == 4.0 ** lvl).all())
    # white_bkgd=False: the plain rgb
    raw = bl.table["images"][:H * W, :3].numpy().astype(np.float32) / np.float32(255)
    assert np.array_equal(bl.image_rays(0)[1].numpy(), raw)


def test_flat_layout_at_16_degrees():
    """The 96-wide flat layout: 618 912 parameters, the pack / unpack round trip, and layers.5.0's [h4, enc] columns at kernel columns
    96..351 and 0..95; the 8-degree table is unchanged."""
    from jnerf_b200.plugin import mip, nerf
    assert mip.REF_LAYERS == mip.ref_layers(8) and mip.REF_LAYERS["layers.0.0"][0] == (256, 48)
    assert mip.kernel_in(8) == nerf.IN and mip.kernel_in(16) == (96, 256, 256, 256, 256, 352, 256, 256, 256, 288, 128)
    wide = mip.ref_layers(16)
    assert wide["layers.0.0"][0] == (256, 96) and wide["layers.5.0"][0] == (256, 352)
    g = torch.Generator().manual_seed(0)
    ref = {name: ((torch.rand((o, i), generator=g) - 0.5).half().float(), (torch.rand(o, generator=g) - 0.5).half().float())
           for name, ((o, i), _, _, _) in wide.items()}
    flat = mip.pack(ref, 16)
    assert flat.numel() == 618912 == nerf.w_offsets(mip.kernel_in(16))[-1]
    for degs in (16, None):
        back = mip.unpack(flat, degs)
        assert all(torch.equal(back[k][0], W) and torch.equal(back[k][1], b) for k, (W, b) in ref.items())
    assert int((flat != 0).sum()) <= sum(W.numel() + b.numel() for W, b in ref.values())
    off = nerf.w_offsets(mip.kernel_in(16))
    W0 = flat[off[0]:off[0] + 256 * 96].view(256, 96).float()
    assert torch.equal(W0, ref["layers.0.0"][0])
    W5 = flat[off[5]:off[5] + 256 * 352].view(256, 352).float()
    assert torch.equal(W5[:, :96], ref["layers.5.0"][0][:, 256:]) and torch.equal(W5[:, 96:], ref["layers.5.0"][0][:, :256])
    # the layers after the skip keep their kernel rows and columns; only their offsets move by the wider layers 0 and 5
    W9 = flat[off[9]:off[9] + 128 * 288].view(128, 288).float()
    assert torch.equal(W9[:, :259], ref["view_layers.0.0"][0][:, :259])
    assert len(mip.unpack(mip.pack({k: v for k, v in ref.items()} | {"layers.0.0": (torch.zeros(256, 48), torch.zeros(256)),
                                                                    "layers.5.0": (torch.zeros(256, 304), torch.zeros(256))}))) == 12


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
# mip_multiscale.cu: the ray kernel (uint8, fp32 images), the encoder (8, 16 degrees); mip_mlp_wide.cu: the forward (with and without saved
# activations), dgrad, wgrad and reduce at 12 encoder groups
@pytest.mark.parametrize("src,n_entries", [("mip_multiscale.cu", 4), ("mip_mlp_wide.cu", 5)])
def test_multiscale_kernels_compile_for_sm90a_without_spills(tmp_path, src, n_entries):
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I",
                        os.path.join(ROOT, "include"), "-fmad=false", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "jnerf_b200", "csrc", src), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == n_entries and len(spills) >= n_entries, r.stderr[-3000:]
    assert all(int(a) == 0 and int(b) == 0 for a, b in spills), r.stderr[-3000:]


def _runner(tmp_path, monkeypatch, cfg_fn="multicam_cfg", **over):
    import multicam_cpu_backend
    fake = multicam_cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as ops
    loss_bwd = ops.mip_composite_loss_bwd
    masks = []

    def spy(raw, t, rays, target, mask, *a, **k):
        masks.append(mask)
        return loss_bwd(raw, t, rays, target, mask, *a, **k)
    monkeypatch.setattr(ops, "mip_composite_loss_bwd", spy)
    from jnerf_b200 import mip_runner, plugin  # noqa: F401
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**getattr(mip_runner, cfg_fn)(seed=1, num_samples=16, log_dir=str(tmp_path), **over))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=4 if split == "train" else 20, H=H, W=W, batch_size=8)
    return mip_runner.MipRunner(), fake, masks


def test_runner_passes_lossmult_as_the_mask(tmp_path, monkeypatch, capsys):
    r, fake, masks = _runner(tmp_path, monkeypatch)
    m = r.model
    assert not m.using_fp16 and m.layers[0][0].in_features == 96 and m.layers[5][0].in_features == 352
    seen = []
    ds = r.dataset["train"]
    nxt = type(ds).__next__

    def record(self):
        b = nxt(self)
        seen.append(b[2].clone())
        return b
    monkeypatch.setattr(type(ds), "__next__", record)
    p0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    losses = [float(r.train_step()) for _ in range(3)]
    assert all(np.isfinite(losses)) and len(masks) == 3
    assert all(torch.equal(a, b) for a, b in zip(masks, seen)) and any(bool((s > 1).any()) for s in seen)
    assert all(not torch.equal(p0[k], v) for k, v in m.state_dict().items())
    psnr = r.test()
    out = capsys.readouterr().out
    assert np.isfinite(psnr) and sorted(r.test_psnr_by_size) == [(4, 3), (8, 6), (16, 12), (32, 24)]
    assert all(f"TEST PSNR {w}x{h}====" in out for w, h in r.test_psnr_by_size) and "TOTAL TEST PSNR====" in out
    assert len(os.listdir(tmp_path / "test" / "test")) == 2 * 8                    # two views at four sizes: render + ground truth

    masks.clear()
    r, _, masks = _runner(tmp_path, monkeypatch, disable_multiscale_loss=True)
    r.train_step()
    assert masks == [None]
    r, _, masks = _runner(tmp_path, monkeypatch, cfg_fn="mip_cfg")
    r.train_step()
    assert masks == [None]


def test_refusals(tmp_path, monkeypatch):
    with pytest.raises(NotImplementedError, match="8 or 16"):
        _runner(tmp_path, monkeypatch, max_deg_point=12)
