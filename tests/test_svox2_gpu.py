"""Plenoxels kernels on the GPU against the fp64 / fp32 restatement of tests/svox_cpu_backend.py, determinism of seeded training with a
resample, learning on the stand-in, and a reference-format ckpt.npz.

Error bound of the training step: per ray |rgb_gpu - rgb_ref| <= 1e-4 (fp32 marching with __expf against fp64).  Per gradient entry
|g_gpu - g_ref| <= 1e-3 * s + n * 2^-49: s is the sum over the n terms the entry received of each term's scale (the operands its fp32
evaluation subtracts or multiplies, svox_cpu_backend.trace), and each fixed-point term is rounded to the nearest 2^-48.  1e-3 covers the
transmittance's drift: log T is a running fp32 sum of up to a few hundred terms.  The scale also carries each weight's own fp32 error,
T (1 - __expf(-pcnt)) losing up to ~2 ulp of T to the cancellation when pcnt is small, and each corner weight the fp32 error of the
sample's position (a factor p or 1 - p near 0 loses its relative accuracy).

Where oracle/_ref/libref_svox.so is built (oracle/svox.mk), the same inputs also go through the reference's own kernels: forward within
fp32 tolerance, gradients (float atomics, so not bit-reproducible) within the same per-entry bound."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import svox_cpu_backend as ref  # noqa: E402

pytestmark = pytest.mark.gpu
OPTS = (0.5, 1e-10, 1e-7, 1.0)


def _grid(n, seed, empty=0.3, device="cuda"):
    """A random sparse grid n^3: a fraction `empty` of the links -1, densities in [0, 40) with some at the 1e-10 threshold, SH ~ N(0, 0.3)."""
    rng = np.random.default_rng(seed)
    keep = rng.random(n ** 3) >= empty
    links = np.full(n ** 3, -1, np.int32)
    cap = int(keep.sum())
    links[keep] = rng.permutation(cap).astype(np.int32)
    dens = (rng.random(cap) * 40).astype(np.float32)
    dens[rng.random(cap) < 0.1] = np.float32(1e-10)
    dens[rng.random(cap) < 0.2] = 0
    sh = (rng.standard_normal((cap, 27)) * 0.3).astype(np.float32)
    return links.reshape(n, n, n), dens, sh


def _cams(n_img, seed):
    from jnerf_b200.plugin.dataset import synthetic_cameras
    m = np.stack(synthetic_cameras(n_img, radius=3.0, seed=seed)).astype(np.float32) @ np.diag(np.array([1, -1, -1, 1], np.float32))
    m[:, :3, 3] *= np.float32(2 / 3)
    return np.ascontiguousarray(m[:, :3, :4].reshape(-1, 12))


XFORM = lambda n: np.array([0.5 * n - 0.5] * 3 + [0.5 * n] * 3, np.float32)      # noqa: E731  radius 1, centre 0


@pytest.mark.parametrize("n", [64, 128])
def test_train_step_against_fp64(n):
    from jnerf_b200 import ops
    links, dens, sh = _grid(n, n)
    W = H = 24
    n_img = 3
    c2w = _cams(n_img, n)
    rng = np.random.default_rng(1)
    images = rng.integers(0, 256, (n_img * H * W, 4), dtype=np.uint8)
    R = 400
    pix = rng.integers(0, n_img * H * W, R).astype(np.int32)
    intr = (6.0, 6.0, W / 2, H / 2)                                   # cameras outside the box, wide enough that corner rays miss it
    cu = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
    gd = torch.zeros(dens.shape[0], dtype=torch.int64, device="cuda")
    gs = torch.zeros(sh.shape, dtype=torch.int64, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    se = ops.svox_train_step(cu(pix), W, H, cu(c2w), intr, cu(images), cu(links), cu(dens), cu(sh), XFORM(n), OPTS, gd, gs, flag)
    torch.cuda.synchronize()
    assert int(flag.item()) == 0
    se_r, gd_r, gs_r, nd, ns, sd, ss = ref.train_step(pix, W, H, c2w, intr, images, links, dens.astype(np.float64), sh.astype(np.float64),
                                                       XFORM(n), OPTS)
    # rays that miss the box and rays that terminate early are both present
    rgb = ref.render(1, 0, W, c2w[0], intr, links, dens.astype(np.float64), sh.astype(np.float64), XFORM(n), OPTS)
    assert np.isfinite(rgb).all()
    out = ops.svox_render(W * H, 0, W, cu(c2w[0]), intr, cu(links), cu(dens), cu(sh), XFORM(n), OPTS).cpu().numpy()
    out_r = ref.render(W * H, 0, W, c2w[0], intr, links, dens.astype(np.float64), sh.astype(np.float64), XFORM(n), OPTS)
    assert np.abs(out - out_r).max() <= 1e-4, np.abs(out - out_r).max()
    assert (np.abs(out_r - 1.0) < 1e-12).all(-1).any() and (np.abs(out_r - 1.0) > 0.1).any()
    assert np.abs(se.cpu().numpy() - se_r).max() <= 1e-3
    assert (nd > 0).sum() > 1000
    for g, g_r, cnt, scale in ((gd.cpu().numpy(), gd_r, nd, sd), (gs.cpu().numpy(), gs_r, ns, ss)):
        g = g.astype(np.float64) / 2.0 ** 48
        tol = 1e-3 * scale + cnt * 2.0 ** -49
        err = np.abs(g - g_r)
        i = np.unravel_index(np.argmax(err / np.maximum(tol, 1e-300)), err.shape)
        assert (err <= tol).all(), ("worst entry", i, g[i], g_r[i], scale[i], cnt[i], (err > tol).sum())
    lib = ref.ref_svox_lib()
    if lib is None:
        return
    # the reference's own kernels: rays as a dataset hands them over, rgb from its forward, the MSE gradient of its backward
    o, d = ref.pixel_rays_f32(pix, W, H, c2w, intr)
    px = images[pix].astype(np.float32) / np.float32(255)
    gt = px[:, :3] * px[:, 3:] + (np.float32(1) - px[:, 3:])
    off, scl = cu(XFORM(n)[:3].copy()), cu(XFORM(n)[3:].copy())
    rgb_ref = torch.empty((R, 3), dtype=torch.float32, device="cuda")
    cap = dens.shape[0]
    args = (cu(o), cu(d), cu(links), n, n, n, cap, cu(dens), cu(sh), off, scl)
    assert lib.ref_svox_render(R, *(a.data_ptr() if torch.is_tensor(a) else a for a in args), rgb_ref.data_ptr(), None) == 0
    gdr = torch.zeros(cap, dtype=torch.float32, device="cuda")
    gsr = torch.zeros((cap, 27), dtype=torch.float32, device="cuda")
    gt_t = cu(np.ascontiguousarray(gt))
    assert lib.ref_svox_backward(R, *(a.data_ptr() if torch.is_tensor(a) else a for a in args), gt_t.data_ptr(), rgb_ref.data_ptr(),
                                 gdr.data_ptr(), gsr.data_ptr(), None) == 0
    torch.cuda.synchronize()
    rgb_ours = ops.svox_render(W * H, 0, W, cu(c2w[0]), intr, cu(links), cu(dens), cu(sh), XFORM(n), OPTS)
    sel = pix < W * H                                                    # the rays of camera 0, rendered by both
    assert np.abs(rgb_ref.cpu().numpy()[sel] - rgb_ours.cpu().numpy()[pix[sel]]).max() <= 1e-4
    for g, g_r, cnt, scale in ((gd.cpu().numpy(), gdr.cpu().numpy(), nd, sd), (gs.cpu().numpy(), gsr.cpu().numpy(), ns, ss)):
        err = np.abs(g.astype(np.float64) / 2.0 ** 48 - g_r)
        assert (err <= 1e-3 * scale + cnt * 2.0 ** -49 + cnt * 1e-7 * scale).all(), err.max()


def test_tv_rmsprop_sample_dilate_compact():
    from jnerf_b200 import ops
    n = 32
    links, dens, sh = _grid(n, 7)
    links[0, 0, 0] = 0
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    G = n ** 3
    for data, ign, scale in ((dens.reshape(-1, 1), False, 1e-5), (sh, True, 1e-3)):
        start, nc = G - 100, 500                                      # wraps around the end of the grid
        g = torch.zeros(data.shape, dtype=torch.int64, device="cuda")
        ops.svox_tv_grad(cu(links), cu(data), start, nc, scale / nc, ign, g, flag)
        g_r = ref.tv_grad(links, data, start, nc, scale / nc, ign)
        err = np.abs(g.cpu().numpy() / 2.0 ** 48 - g_r)
        assert (err <= 1e-5 * np.abs(g_r).max() + 4 * 2.0 ** -49).all(), err.max()
    assert int(flag.item()) == 0
    # RMSprop: fixed-point gradient in, fp32 update out, gradient cleared
    rng = np.random.default_rng(3)
    p, v = rng.standard_normal(1000).astype(np.float32), rng.random(1000).astype(np.float32)
    g = rng.integers(-2 ** 50, 2 ** 50, 1000)
    ps, vs = rng.standard_normal(2700).astype(np.float32), rng.random(2700).astype(np.float32)
    gsh = rng.integers(-2 ** 40, 2 ** 40, 2700)
    tp, tv, tg, tps, tvs, tgs = (cu(a) for a in (p, v, g, ps, vs, gsh))
    ops.svox_rmsprop(tp, tps, tg, tgs, tv, tvs, 30.0, 0.01, 0.95, 0.9, 1e-8)
    for a, b, gg, vv, lr, al in ((tp, p, g, v, 30.0, 0.95), (tps, ps, gsh, vs, 0.01, 0.9)):
        pr, _ = ref.rmsprop(b, vv, (gg.astype(np.float64) / 2.0 ** 48).astype(np.float32), lr, al, 1e-8)
        np.testing.assert_allclose(a.cpu().numpy(), pr, rtol=2e-6, atol=2e-6 * np.abs(pr).max())
    assert int(tg.abs().sum()) == 0 and int(tgs.abs().sum()) == 0
    # sample: bit-exact
    pts = (rng.random((5000, 3)) * (n + 2) - 1.5).astype(np.float32)
    d, s = ops.svox_sample(cu(pts), cu(links), cu(dens), cu(sh), True)
    d_r, s_r = ref.sample(pts, links, dens, sh, True)
    assert np.array_equal(d.cpu().numpy(), d_r) and np.array_equal(s.cpu().numpy(), s_r)
    # dilate and compact: identical masks, links and capacity
    mask = (rng.random((n, n, n)) < 0.01).astype(np.uint8)
    m1 = ops.svox_dilate(cu(mask))
    assert np.array_equal(m1.cpu().numpy(), ref.dilate(mask))
    dense = rng.random((n, n, n)).astype(np.float32)
    lattice = np.array([-0.25, -0.25, -0.25, 0.5, 0.5, 0.5], np.float32)
    cap = int(m1.sum())
    lk, dd, pp = ops.svox_compact(m1, cu(dense), lattice, cap)
    lk_r, dd_r, pp_r = ref.compact(m1.cpu().numpy(), dense, lattice)
    assert np.array_equal(lk.cpu().numpy(), lk_r) and np.array_equal(dd.cpu().numpy(), dd_r) and np.array_equal(pp.cpu().numpy(), pp_r)


def test_weight_render_against_fp64():
    from jnerf_b200 import ops
    n = 32
    rng = np.random.default_rng(5)
    data = (rng.random((n, n, n)) * 3).astype(np.float32)
    data[rng.random((n, n, n)) < 0.5] = 0
    c2w = _cams(1, 9)[0]
    intr = (20.0, 20.0, 8.0, 8.0)
    out = torch.zeros((n, n, n), dtype=torch.float32, device="cuda")
    ops.svox_weight_render(torch.from_numpy(data).cuda(), 16, 16, torch.from_numpy(c2w).cuda(), intr, XFORM(n), 0.5, 0.2, out)
    out_r = ref.weight_render(data, 16, 16, c2w, intr, XFORM(n), 0.5, 0.2, np.zeros((n, n, n)))
    assert (out_r > 0).sum() > 100
    # a ray whose transmittance reaches the stop threshold (0.2) within fp32 rounding may stop one sample earlier or later than in fp64;
    # every other cell agrees to 1e-5
    bad = np.abs(out.cpu().numpy() - out_r) > 1e-5
    assert bad.sum() <= 2e-3 * (out_r > 0).sum(), (bad.sum(), (out_r > 0).sum())


def _small_runner(tmp_path, seed_over=None):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.svox2_runner import Svox2Runner, svox2_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    c = svox2_cfg(synthetic=True, reso_list=[[64] * 3, [128] * 3], batch_size=5000, epoch_size=40, upsamp_every=80, n_iters=160, log_dir=str(tmp_path),
                  max_grid_elements=44000000)
    for s in ("train", "test"):
        c["dataset"][s].update(n_images=20, H=64, W=64, epoch_size=40 * 5000)
    update_cfg(**c)
    return Svox2Runner()


def test_determinism_and_learning(tmp_path):
    """Two seeded runs of 160 steps with one resample (64^3 -> 128^3) on the 64x64 stand-in give identical bytes.  The test PSNR is the
    mean over the stand-in's 2 test views; measured on an H100 80GB HBM3 (700 W): 7.5 dB before training, 20.4 dB after."""
    outs = []
    for k in range(2):
        r = _small_runner(tmp_path / str(k))
        if k == 0:
            psnr0 = r.test()
        r.train()
        g = r.model
        outs.append((g.density_data.cpu().numpy().tobytes(), g.sh_data.cpu().numpy().tobytes(), g._links.cpu().numpy().tobytes()))
        if k == 0:
            assert g._links.shape == (128, 128, 128)
            psnr1 = r.test()
    print(f"svox2 learning: test PSNR {psnr0:.2f} -> {psnr1:.2f} dB")
    assert outs[0] == outs[1]
    assert psnr1 > psnr0 + 5.0, (psnr0, psnr1)


def test_reference_format_ckpt_renders_the_same_image(tmp_path):
    from jnerf_b200.plugin.svox2 import Camera, SparseGrid
    links, dens, sh = _grid(64, 11)
    g = SparseGrid(64, use_sphere_bound=False)
    g._links, g.density_data, g.sh_data = torch.from_numpy(links).cuda(), torch.from_numpy(dens).cuda().view(-1, 1), torch.from_numpy(sh).cuda()
    g.capacity = dens.shape[0]
    np.savez(tmp_path / "ckpt.npz", radius=np.ones(3, np.float32), center=np.zeros(3, np.float32), links=links, density_data=dens.reshape(-1, 1),
             sh_data=sh.astype(np.float16), basis_type=1)
    h = SparseGrid.load(str(tmp_path / "ckpt.npz"))
    cam = Camera(torch.from_numpy(_cams(1, 4)[0]).cuda(), 40.0, 40.0, 24.0, 24.0, 48, 48)
    a, b = g.volume_render_image(cam).cpu().numpy(), h.volume_render_image(cam).cpu().numpy()
    # fp16 SH: relative rounding 2^-11 of coefficients |c| < 2, through 9 basis values <= 1.1 per channel
    assert np.abs(a - b).max() <= 9 * 1.1 * 2 * 2.0 ** -11
    assert np.array_equal(h._links.cpu().numpy(), links)
