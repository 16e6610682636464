"""LLFFDataset (forward-facing captures in the `poses_bounds.npy` layout, llff_dataset.py of the reference) without a GPU: the pose
pipeline against a numpy restatement written here, the in-memory image reduction, the hold-out split, the synthetic stand-in's
consistency under the loader's similarity transform, the reference's own ngp_llff.py through init_cfg on the CPU backend at seven
occupancy cascades, and the hash table at aabb_scale 64 / 32."""
import math
import os
import re

import numpy as np
import pytest
import torch

import oracle_lib as ol
from jnerf_b200.plugin import dataset as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G3 = 128 ** 3


@pytest.fixture()
def cpu_device(monkeypatch):
    monkeypatch.setattr(D, "DEVICE", "cpu")


def _reference_tree():
    """$NGP_REF, else the default oracle/Makefile builds the reference sources from."""
    if os.environ.get("NGP_REF"):
        return os.environ["NGP_REF"]
    m = re.search(r"^NGP_REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M)
    return m.group(1) if m else ""


# ------------------------------------------------------------------------------------------------ helpers shared with test_llff_gpu.py
def update_bitfield(grid, mean, cascades):
    """orc_update_bitfield with a bitfield sized for `cascades` levels."""
    bits = np.zeros(G3 * cascades // 8, np.uint8)
    ol.oracle().orc_update_bitfield(ol._ptr(grid), ol._f32(mean), ol._u32(cascades), ol._ptr(bits))
    return bits


def shells_bitfield(cascades, seed=0):
    """An occupancy grid with occupied cells in EVERY cascade, the outermost included: in cascade k (cube of side 2^k around the
    centre) a spherical shell of radius 0.36 * 2^k plus a sprinkle of random cells; built through the oracle's bitfield path (so
    every coarser cascade also holds the max-pool of the finer one).  Returns (bitfield, density grid)."""
    rng = np.random.default_rng(seed)
    grid = np.zeros(G3 * cascades, np.float32)
    ids = np.arange(G3, dtype=np.uint32)

    def minv(x):
        x = x & 0x49249249
        x = (x | (x >> 2)) & 0xc30c30c3
        x = (x | (x >> 4)) & 0x0f00f00f
        x = (x | (x >> 8)) & 0xff0000ff
        x = (x | (x >> 16)) & 0x0000ffff
        return x
    c = [((minv(ids >> k) + 0.5) / 128 - 0.5) for k in range(3)]
    r = np.sqrt(c[0] ** 2 + c[1] ** 2 + c[2] ** 2)                   # in units of the cascade's side
    for lvl in range(cascades):
        occ = (np.abs(r - 0.36) < 0.02) | (rng.random(G3) < 2e-4)
        grid[lvl * G3:(lvl + 1) * G3] = np.where(occ, 1.0, 0.0)
    return update_bitfield(grid, 1.0, cascades), grid


def wide_rays(R, cascades, seed=0):
    """Rays for a `cascades`-level grid: a third start inside the unit cube, a third between the unit cube and the aabb, a third far
    outside the aabb looking in."""
    rng = np.random.default_rng(seed)
    half = 2.0 ** (cascades - 1) / 2
    v = rng.normal(size=(R, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    dist = np.where(np.arange(R) % 3 == 0, rng.uniform(0.0, 0.45, R), np.where(np.arange(R) % 3 == 1, rng.uniform(0.6, half, R), rng.uniform(1.8 * half, 3 * half, R)))
    o = 0.5 + dist[:, None] * v
    tgt = 0.5 + rng.uniform(-0.3, 0.3, size=(R, 3)) * np.where(np.arange(R) % 2 == 0, 1.0, half)[:, None]
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


def ref_llff(poses_bounds, hw, factor, bd_factor=.75, recenter=True, llffhold=0, correct_pose=(1, -1, -1)):
    """llff_dataset.py:136-196,221-223,376-383 restated with numpy: (n,17) file contents and the loaded image size -> the NGP 3x4
    transforms of all views, focal length, test indices, and the similarity (scale, mean camera) applied to the cameras."""
    n = poses_bounds.shape[0]
    P = poses_bounds[:, :15].reshape(n, 3, 5).astype(np.float64).copy()
    bds = poses_bounds[:, 15:].astype(np.float32)
    P[:, 0, 4], P[:, 1, 4] = hw[0], hw[1]
    P[:, 2, 4] = P[:, 2, 4] / factor
    P = np.stack([P[:, :, 1], -P[:, :, 0], P[:, :, 2], P[:, :, 3], P[:, :, 4]], 2).astype(np.float32)
    sc = np.float32(1.0) / (bds.min() * np.float32(bd_factor))
    P[:, :, 3] *= sc

    def avg(P):
        z = P[:, :, 2].sum(0)
        z = z / np.linalg.norm(z)
        up = P[:, :, 1].sum(0)
        x = np.cross(up, z)
        x = x / np.linalg.norm(x)
        y = np.cross(z, x)
        y = y / np.linalg.norm(y)
        return np.stack([x, y, z, P[:, :, 3].mean(0)], 1)
    A = np.eye(4)
    if recenter:
        A[:3] = avg(P)
        full = np.tile(np.eye(4), (n, 1, 1))
        full[:, :3] = P[:, :, :4]
        P[:, :, :4] = (np.linalg.inv(A) @ full)[:, :3].astype(np.float32)
    if llffhold > 0:
        i_test = list(range(0, n, llffhold))
    else:
        i_test = [int(np.argmin(((avg(P)[:, 3] - P[:, :, 3]) ** 2).sum(-1)))]
    xf = []
    for k in range(n):
        m = P[k, :, :4].copy()
        for c in range(3):
            m[:, c] *= correct_pose[c]
        m[:, 3] = m[:, 3] * np.float32(0.33) + np.float32(0.5)
        xf.append(m[[1, 2, 0]])
    return np.stack(xf), float(P[0, 2, 4]), i_test, float(sc), A


def write_random_llff(root, n, H, W, rng, sub="images_4", ext="png"):
    from PIL import Image
    os.makedirs(os.path.join(root, sub), exist_ok=True)
    rows, imgs = [], []
    for k in range(n):
        m = np.zeros((3, 5))
        m[:, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        m[:, 3] = rng.standard_normal(3) * 3
        m[:, 4] = (H * 4, W * 4, 812.5)
        rows.append(np.concatenate([m.reshape(-1), [rng.uniform(1.0, 2.0), rng.uniform(20.0, 90.0)]]))
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, sub, f"im_{k:03d}.{ext}"))
        imgs.append(img)
    arr = np.stack(rows)
    np.save(os.path.join(root, "poses_bounds.npy"), arr)
    return arr, np.stack(imgs)


# ------------------------------------------------------------------------------------------------ 1. pose pipeline and split
@pytest.mark.parametrize("llffhold", [0, 8])
def test_llff_dataset_against_numpy_restatement(tmp_path, cpu_device, llffhold):
    rng = np.random.default_rng(3)
    n, H, W = 19, 12, 20
    arr, imgs = write_random_llff(str(tmp_path), n, H, W, rng)
    open(tmp_path / "images_4" / "notes.txt", "w").write("not an image")              # other files in the directory are not views
    xf_ref, focal, i_test, _, _ = ref_llff(arr, (H, W), 4, llffhold=llffhold)
    assert i_test == ([0, 8, 16] if llffhold else i_test) and len(i_test) == (3 if llffhold else 1)
    sets = {}
    for mode in ("train", "val", "test"):
        ds = D.LLFFDataset(str(tmp_path), 64, mode=mode, factor=4, llffhold=llffhold, aabb_scale=64, scale=7.0, offset=[1, 2, 3], have_img=False,
                           spherify=True)
        sel = [i for i in range(n) if i not in i_test] if mode == "train" else i_test
        sets[mode] = list(ds.i_select)
        assert sets[mode] == sel and ds.n_images == len(sel)
        assert ds.scale == 0.33 and ds.offset == [0.5, 0.5, 0.5]                        # the arguments are discarded (llff_dataset.py:24-25)
        got = ds.transforms_gpu.numpy().reshape(len(sel), 4, 3).transpose(0, 2, 1)      # stored column-major (llff_dataset.py:127-128)
        assert np.abs(got - xf_ref[sel]).max() <= 1e-6
        assert ds.resolution == [W, H] and (ds.H, ds.W) == (H, W)
        assert np.array_equal(ds.focal_lengths.numpy(), np.full((len(sel), 2), np.float32(812.5 / 4)))
        assert np.array_equal(ds.principal.numpy(), np.full((len(sel), 2), 0.5, np.float32))
        assert np.array_equal(ds.metadata.numpy()[:, [0, 1, 2, 3, 8, 9, 10]], np.zeros((len(sel), 7), np.float32))
        assert ds.aabb_scale == 64 and ds.aabb_range == (-31.5, 32.5)
        assert ds.image_data.dtype == torch.uint8 and ds.image_data.shape == (len(sel), H * W, 4)
        assert np.array_equal(ds.image_data.numpy()[:, :, :3].reshape(len(sel), H, W, 3), imgs[sel]) and bool((ds.image_data[:, :, 3] == 255).all())
        for p, k in zip(ds.poses, sel):                                                 # NeRF camera-to-world before the NGP step
            assert np.abs(D.matrix_nerf2ngp(p, 0.33, [0.5] * 3) - xf_ref[k]).max() <= 1e-6
    assert sets["val"] == sets["test"] and sorted(sets["train"] + sets["test"]) == list(range(n))
    assert D.LLFFDataset(str(tmp_path), 64, mode="test", factor=4).aabb_scale == 32     # llff_dataset.py:32-34
    flipped = D.LLFFDataset(str(tmp_path), 64, mode="test", factor=4, llffhold=8, correct_pose=(1, 1, -1))
    got = flipped.transforms_gpu.numpy().reshape(3, 4, 3).transpose(0, 2, 1)
    assert np.abs(got - ref_llff(arr, (H, W), 4, llffhold=8, correct_pose=(1, 1, -1))[0][[0, 8, 16]]).max() <= 1e-6


def test_batches_come_from_the_selected_views(tmp_path, cpu_device):
    """_RayBatcher on an LLFFDataset: shuffled pixel ids address (view, pixel) of the split, colours are the stored bytes / 255."""
    rng = np.random.default_rng(5)
    arr, imgs = write_random_llff(str(tmp_path), 9, 6, 8, rng)
    ds = D.LLFFDataset(str(tmp_path), 40, mode="train", factor=4, llffhold=4, seed=2)
    pix = ds.next_pixels().numpy()
    assert pix.shape == (40,) and pix.max() < ds.n_images * 48 and len(set(pix.tolist())) == 40
    rgba = ds.rgba_for(torch.from_numpy(pix)).numpy()
    sel = np.array(ds.i_select)
    want = imgs[sel].reshape(-1, 3)[pix].astype(np.float32) / 255
    assert np.array_equal(rgba[:, :3], want) and bool((rgba[:, 3] == 1).all())


# ------------------------------------------------------------------------------------------------ 2. images_{factor} missing
def test_missing_reduced_images_are_reduced_in_memory(tmp_path, cpu_device):
    rng = np.random.default_rng(7)
    H, W, f = 24, 40, 4
    arr, imgs = write_random_llff(str(tmp_path), 5, H, W, rng, sub="images", ext="jpg.png")
    before = sorted((r, tuple(sorted(d)), tuple(sorted(fs))) for r, d, fs in os.walk(tmp_path))
    ds = D.LLFFDataset(str(tmp_path), 16, mode="train", factor=f, llffhold=5)
    assert sorted((r, tuple(sorted(d)), tuple(sorted(fs))) for r, d, fs in os.walk(tmp_path)) == before      # no images_4, no split.json
    assert ds.resolution == [W // f, H // f] and ds.n_images == 4
    box = imgs[1:].reshape(4, H // f, f, W // f, f, 3).astype(np.float64).mean((2, 4))
    got = ds.image_data.numpy()[:, :, :3].reshape(4, H // f, W // f, 3).astype(np.float64)
    assert np.abs(got - box).max() <= 1.0                                                                    # 8-bit rounding of the box mean
    assert np.allclose(ds.focal_lengths.numpy(), 812.5 / f)
    odd = D.LLFFDataset(str(tmp_path), 16, mode="test", factor=7, llffhold=5)                                # (round(H / 7), round(W / 7))
    assert odd.resolution == [int(round(W / 7)), int(round(H / 7))]


# ------------------------------------------------------------------------------------------------ 3. errors
def test_errors(tmp_path, cpu_device):
    rng = np.random.default_rng(9)
    arr, _ = write_random_llff(str(tmp_path), 6, 8, 8, rng)
    os.remove(tmp_path / "images_4" / "im_005.png")
    with pytest.raises(ValueError, match=r"5 images.*6 poses"):
        D.LLFFDataset(str(tmp_path), 16, factor=4)
    with pytest.raises(ValueError, match="factor"):
        D.LLFFDataset(str(tmp_path), 16, factor=None)


# ------------------------------------------------------------------------------------------------ 4. the stand-in is consistent
def test_stand_in_images_agree_with_the_loaded_poses(tmp_path, cpu_device):
    """write_synthetic_llff then LLFFDataset: the loader moves all cameras by one similarity transform (scale 1 / (0.75 * nearest
    bound), then into the mean camera's frame), so a ray of a loaded pose mapped back through it hits the analytic scene at the
    colour stored in the image."""
    H, W, n = 36, 48, 7
    mats = D.write_synthetic_llff(str(tmp_path), n_images=n, H=H, W=W, seed=4)
    assert sorted(os.listdir(tmp_path)) == ["images", "poses_bounds.npy"] and len(os.listdir(tmp_path / "images")) == n
    arr = np.load(tmp_path / "poses_bounds.npy")
    assert arr.shape == (n, 17) and (arr[:, 15] > 0.5).all() and (arr[:, 16] > 4 * arr[:, 15]).all()
    # forward-facing: the baseline is small against the distance to the scene, and all cameras look the same way
    pos = mats[:, :, 3]
    assert np.linalg.norm(pos - pos.mean(0), axis=1).max() < 0.3 * np.linalg.norm(pos.mean(0))
    assert (mats[:, :, 2] @ mats[0, :, 2] > 0.85).all()
    assert np.allclose(arr[:, :15].reshape(n, 3, 5)[:, :, 1], mats[:, :, 0]) and np.allclose(arr[:, :15].reshape(n, 3, 5)[:, :, 0], -mats[:, :, 1])
    ds = D.LLFFDataset(str(tmp_path), 64, mode="train", factor=1, llffhold=3, aabb_scale=64)
    _, focal, i_test, sc, A = ref_llff(arr, (H, W), 1, llffhold=3)
    assert ds.resolution == [W, H] and abs(ds._focal[0] - 0.81 * W) < 1e-4 and bool((ds.image_data[:, :, 3] == 255).all())
    scene = object.__new__(D.SyntheticNerfDataset)
    scene.scale, scene.obj_scale, scene.backdrop_radius = D.NERF_SCALE, 2.2, 8.0
    rng = np.random.default_rng(0)
    checked = 0
    for k in (0, ds.n_images - 1):
        xf = ds.transforms_gpu[k].numpy().reshape(4, 3).T.astype(np.float64)           # NGP 3x4 of the loaded pose
        v, u = rng.integers(2, H - 2, 40), rng.integers(2, W - 2, 40)
        d_cam = np.stack([(u + 0.5 - W / 2) / ds._focal[0], (v + 0.5 - H / 2) / ds._focal[1], np.ones(40)], -1)
        d_ngp = d_cam @ xf[:, :3].T
        # NGP -> loaded NeRF world (undo the axis cycle, offset and scale) -> the writer's world (mean camera frame, then 1 / sc)
        o_w = A[:3, :3] @ ((xf[:, 3] - 0.5) / 0.33)[[2, 0, 1]] + A[:3, 3]
        d_w = d_ngp[:, [2, 0, 1]] @ A[:3, :3].T
        o0 = (o_w / sc * 0.33)[[1, 2, 0]] + 0.5                                         # the writer's NGP coordinates
        d0 = d_w[:, [1, 2, 0]]
        d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
        rgba = scene.shade(torch.from_numpy(np.tile(o0, (40, 1)).astype(np.float32)), torch.from_numpy(d0.astype(np.float32))).numpy()
        stored = ds.image_data[k].numpy().reshape(H, W, 4)[v, u, :3].astype(np.float32) / 255
        err = np.abs(rgba[:, :3] - stored).max(1)
        # a pixel on a texture or silhouette edge may fall on the other side after the round trip in fp32: most agree to 8-bit rounding
        assert (err <= 1.5 / 255).mean() >= 0.9 and np.median(err) <= 1.0 / 255, err
        checked += 40
    assert checked == 80


def test_stand_in_writes_reduced_images_too(tmp_path, cpu_device):
    D.write_synthetic_llff(str(tmp_path), n_images=3, H=32, W=48, factor=4, seed=1)
    assert sorted(os.listdir(tmp_path)) == ["images", "images_4", "poses_bounds.npy"]
    a = D.LLFFDataset(str(tmp_path), 16, mode="train", factor=4, llffhold=3)
    os.rename(tmp_path / "images_4", tmp_path / "elsewhere")
    b = D.LLFFDataset(str(tmp_path), 16, mode="train", factor=4, llffhold=3)            # reduced in memory by the same filter
    assert a.resolution == [12, 8] and torch.equal(a.image_data, b.image_data) and torch.equal(a.transforms_gpu, b.transforms_gpu)


# ------------------------------------------------------------------------------------------------ 5. the reference's ngp_llff.py
def test_reference_ngp_llff_config_builds_and_steps_at_seven_cascades(tmp_path, monkeypatch):
    ref_cfg = os.path.join(_reference_tree(), "projects", "ngp", "configs", "ngp_llff.py")
    if not os.path.exists(ref_cfg):
        pytest.skip("reference tree not present")
    import cpu_backend
    fake = cpu_backend.install(monkeypatch)
    monkeypatch.setattr(D, "DEVICE", "cpu")
    monkeypatch.setattr(ol, "update_bitfield", lambda grid, mean, cascades=5: update_bitfield(grid, mean, cascades))
    monkeypatch.setenv("NGP_PIPELINE", "0")
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.utils.config import get_cfg, init_cfg
    monkeypatch.chdir(tmp_path)
    D.write_synthetic_llff(os.path.join("data", "fern"), n_images=9, H=96, W=128, seed=2)      # images/ only: reduced 8x at load time
    get_cfg().clear()
    init_cfg(ref_cfg)                                                                           # the file itself, unchanged
    cfg = get_cfg()
    ns = {}
    exec(open(ref_cfg).read(), ns)
    ref = {k: v for k, v in ns.items() if not k.startswith("__")}
    assert R.llff_cfg("data/fern") == ref
    mine = R.llff_cfg("/some/capture", n_rays_per_batch=8)
    assert mine["dataset"]["val"]["root_dir"] == "/some/capture" and mine["dataset_dir"] == "/some/capture" and mine["n_rays_per_batch"] == 8
    cfg.n_rays_per_batch, cfg.target_batch_size = 48, 32768                                      # the scalar oracle marches these in milliseconds
    r = R.Runner()
    s, ds = r.sampler, r.dataset["train"]
    assert isinstance(ds, D.LLFFDataset) and ds.n_images == 7 and ds.resolution == [16, 12] and r.dataset["val"].n_images == 2
    assert s.NERF_CASCADES == 7 and s.max_cascade == 6 and s.aabb_range == (-31.5, 32.5) and s.const_dt is False
    assert s.density_grid.numel() == 7 * G3 and s.density_grid_bitfield.numel() == 7 * G3 // 8
    assert r.fast and r.model.pos_encoder.levels.n_params == r.model.pos_encoder.m_grid.numel()  # the fused path, not the per-operator step
    # one occupancy-grid update over max_cascade + 1 = 7 levels (a small sample count instead of the 14.7 M of a real one)
    fake.calls.clear()
    s.update_density_grid_nerf(0.95, 40000, 0)
    assert fake.calls == ["grid_mark_untrained", "grid_generate_samples", "density_fwd", "grid_splat", "grid_ema", "grid_update_bitfield"]
    per = s.density_grid.reshape(7, G3)
    assert all(int((per[k] > 0).sum()) > 0 for k in range(7))                                     # samples landed in every cascade
    assert all(int(s.density_grid_bitfield.reshape(7, -1)[k].count_nonzero()) > 0 for k in range(7))
    cfg.m_training_step = 1
    fake.calls.clear()
    losses = [float(r.train_step().mean()) for _ in range(3)]
    assert fake.calls[:6] == ["prepare_batch", "march", "compact", "network_fwd", "composite_loss_bwd", "network_bwd"]
    assert all(np.isfinite(losses)) and int(s.n_samples_dev.item()) > 0
    o, d = r.pose_rays(ds.poses[0])                                                               # Runner.pose_rays on an LLFF pose
    o2, d2 = ds.generate_rays_total_test(0)
    assert torch.equal(o, o2) and torch.allclose(d, d2, atol=1e-6)


# ------------------------------------------------------------------------------------------------ 6. hash table at aabb_scale 64 / 32
@pytest.mark.parametrize("aabb_scale", [64, 32])
def test_hash_table_layout_of_wide_scenes(aabb_scale, monkeypatch):
    import cpu_backend
    cpu_backend.install(monkeypatch)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.plugin.encoders import HashEncoder
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(fp16=True, hash_func="p0 ^ p1 * 19349663 ^ p2 * 83492791", dataset_obj=type("DS", (), {"aabb_scale": aabb_scale})())
    enc = HashEncoder()
    # grid_encode.py:19-36 restated: python doubles, 8-aligned level sizes capped at 2^19 entries
    pls = math.exp(math.log(2048 * aabb_scale / 16) / 15)
    offsets, off = [], 0
    for i in range(16):
        res = int(math.ceil(2.0 ** (i * math.log2(pls)) * 16 - 1.0)) + 1
        offsets.append(off)
        off += min((res ** 3 + 7) // 8 * 8, 1 << 19)
    offsets.append(off)
    cfg = ol.HashCfg(aabb_scale)
    lv = enc.levels
    assert lv.per_level_scale == pls == cfg.per_level_scale
    assert list(lv.offsets) == offsets == list(cfg.offsets)
    assert enc.m_grid.numel() == 2 * off and enc.m_grid.dtype == torch.float16
    dense = [i for i in range(16) if offsets[i + 1] - offsets[i] < (1 << 19)]
    assert dense == [0, 1, 2] and round(16 * pls ** 15) == 2048 * aabb_scale            # three dense levels; finest resolution 131 072 at 64
