"""Depth maps of the whole-frame renderer on the H100 (ngp_render_composite_round_depth), on the lego and fox stand-ins trained a few
hundred steps as in test_render_gpu.py and on a small fp16 vanilla-NeRF runner: the colour outputs do not move when depth is asked
for, each ray's sum(w t) against an fp64 recomposition of the same samples with a per-ray bound of the fp32 sequential sum, the
early-stopping bound on the sum, the depth of a trained lego stand-in against the analytic hit distance, and the spiral path on the
trained forward-facing stand-in."""
import os

import numpy as np
import pytest
import torch

from test_render_gpu import _runner

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                                                          # unit roundoff of fp32
MIN_CONE = np.sqrt(3.0) / 1024.0


def _nerf_runner():
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.nerf_runner import NerfRunner
    from jnerf_b200.runner import nerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**nerf_cfg(fp16=True, synthetic=True, seed=5, optim=dict(type="Adam", lr=5e-4, eps=1e-15, betas=(0.9, 0.99))))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 8
    cfg.dataset.train.H = cfg.dataset.train.W = 96
    cfg.dataset.val = None
    r = NerfRunner()
    assert not r.fast and r.model.using_fp16
    r.train(200)
    torch.cuda.synchronize()
    return r


@pytest.fixture(scope="module")
def runners():
    return {}


@pytest.fixture(params=["lego", "fox", "nerf"])
def runner(request, runners):
    if request.param not in runners:
        runners[request.param] = _nerf_runner() if request.param == "nerf" else _runner(request.param)
    return runners[request.param]


def render(r, o, d, eps, rng, depth):
    """Runner.render_rays from the sampler rng state `rng`, which is left as it was."""
    s = r.sampler
    keep = s.rng.copy()
    s.rng[:] = rng
    out = r.render_rays(o, d, eps, depth=True) if depth else r.render_rays(o, d, eps)
    s.rng[:] = keep
    return out


def frame(r, img_id):
    return r.dataset["train"].generate_rays_total_test(img_id)


def test_colour_outputs_do_not_move_with_depth(runner):
    r = runner
    o, d = frame(r, 2)
    rng = r.sampler.rng.copy()
    for eps in (0.0, 1e-4):
        rgb, alpha, n, rounds = render(r, o, d, eps, rng, False)
        rgb1, alpha1, n1, rounds1, S = render(r, o, d, eps, rng, True)
        assert torch.equal(rgb, rgb1) and torch.equal(alpha, alpha1) and torch.equal(n, n1) and rounds == rounds1
        assert S.shape == (o.shape[0],) and S.dtype == torch.float32 and torch.isfinite(S).all()
        assert (S >= 0).all() and (S[n == 0] == 0).all() and (S > 0).sum() > 1000


def slab_exit(o, d, lo, hi):
    """fp64 exit distance of each ray from the box [lo, hi]^3 (t at which it leaves; meaningful for rays that meet the box)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0, t1 = (lo - o) * inv, (hi - o) * inv
    return np.nanmin(np.maximum(t0, t1), axis=1)


def reference_sums(r, o, d, rng):
    """Per ray, from ngp_march's samples under render_rays' jitter layout and the model's network on them: the fp64 recomposition
    sum(w t) (t recovered in fp64 from the warped positions) and a bound on |fp32 sequential sum - fp64| built from the per-sample
    error of the fp32 alpha (__expf, the dt product), of the transmittance product, of the recovered t and of the fp32 accumulation."""
    from jnerf_b200 import ops
    s = r.sampler
    tile, C = int(r.cfg.n_rays_per_batch), s.NERF_CASCADES
    lo, hi = (float(v) for v in s.aabb_range)
    diag = hi - lo
    st = rng.copy()
    out = torch.empty((s.max_samples, 4), dtype=torch.float16, device="cuda")
    ref, bound = np.zeros(o.shape[0]), np.zeros(o.shape[0])
    mx = MIN_CONE * (1 << (C - 1))
    for p in range(0, o.shape[0], tile):
        oo, dd = o[p:p + tile].contiguous(), d[p:p + tile].contiguous()
        coords, _, numsteps, counters = ops.march(oo, dd, s.density_grid_bitfield, s.aabb_range, s.max_samples, s.cone_angle_constant,
                                                  s.near_distance, C, s.const_dt, st)
        ops.pcg32_advance(st)
        r._net_infer(coords, counters[1:2], out)
        total = int(counters[1].item())
        c = coords[:total].double().cpu().numpy()
        net = out[:total].double().cpu().numpy()
        ns = numsteps.view(torch.int32).cpu().numpy().astype(np.int64)
        o64, d64 = oo.double().cpu().numpy(), dd.double().cpu().numpy()
        for k in range(ns.shape[0]):
            cnt, base = ns[k]
            if cnt == 0:
                continue
            rows = slice(base, base + cnt)
            pos = c[rows, :3] * diag + lo
            t = ((pos - o64[k]) @ d64[k]) / (d64[k] @ d64[k])
            dt = c[rows, 3] * (mx - MIN_CONE) + MIN_CONE
            sig = net[rows, 3]
            y = np.exp(sig) * dt
            alpha = -np.expm1(-y)
            T = np.concatenate([[1.0], np.cumprod(1.0 - alpha)[:-1]])
            w = alpha * T
            ref[p + k] = (w * t).sum()
            # |alpha32 - alpha|: __expf of -y (2^-22 absolute), y's relative error (__expf(sig): 2^-22 + |sig| 2^-23 for the exponent's
            # rounding, the unwarped dt and the product: 2^-22) times dalpha/dlog y = y e^-y <= 1/e, and the final subtraction
            e_a = 4 * U + y * np.exp(-y) * (4 * U + np.abs(sig) * 2 * U + 4 * U) + U
            e_T = np.concatenate([[0.0], np.cumsum(e_a)[:-1]]) + np.arange(cnt) * U * T
            e_w = e_a * T + alpha * e_T + U * w
            e_t = 4 * U * (diag + np.abs(pos).max(1)) / np.sqrt(d64[k] @ d64[k])          # the warped position's and p's rounding
            bound[p + k] = (e_w * t).sum() + (w * e_t).sum() + (cnt + 1) * U * ref[p + k] * 1.01
    return ref, bound


def test_sum_matches_fp64_recomposition(runner, request):
    r = runner
    o, d = frame(r, 2)
    rng = r.sampler.rng.copy()
    _, _, n, _, S = render(r, o, d, 0.0, rng, True)
    ref, bound = reference_sums(r, o, d, rng)
    S = S.double().cpu().numpy()
    err = np.abs(S - ref)
    hit = n.cpu().numpy() > 0
    assert hit.sum() > 1000
    rel = (err / np.maximum(bound, 1e-30))[hit]
    print(f"{request.node.name}: sum(w t) vs fp64, {int(hit.sum())} rays: max |err| {err.max():.3e}, max err / bound {rel.max():.3f}, "
          f"median bound {np.median(bound[hit]):.3e}")
    assert (err <= bound).all(), (err.max(), np.argmax(err - bound))
    assert (S[~hit] == 0).all() and (ref[~hit] == 0).all()


def test_early_stopping_bound_on_the_sum(runner):
    r = runner
    o, d = frame(r, 3)
    rng = r.sampler.rng.copy()
    eps = 1e-4
    _, _, n0, _, S0 = render(r, o, d, 0.0, rng, True)
    _, _, n1, _, S1 = render(r, o, d, eps, rng, True)
    lo, hi = (float(v) for v in r.sampler.aabb_range)
    t_exit = slab_exit(o.double().cpu().numpy(), d.double().cpu().numpy(), lo, hi)
    S0, S1 = S0.double().cpu().numpy(), S1.double().cpu().numpy()
    n0 = n0.cpu().numpy()
    hit = n0 > 0
    # the stopped ray lost samples whose weights sum to at most T < eps, each at t <= t_exit; the shared prefix is bit-identical, so
    # the rest is the rounding of the fp32 sums and of the transmittance
    rnd = (n0 + 1) * 2 * U * S0 + eps * t_exit * n0 * 2 * U
    diff = np.abs(S1 - S0)
    assert (diff[hit] <= eps * t_exit[hit] + rnd[hit]).all(), (diff[hit] - eps * t_exit[hit] - rnd[hit]).max()
    assert (n1.cpu().numpy() <= n0).all() and (S1[~hit] == 0).all()


# ------------------------------------------------------------------------------------------------ geometry on a trained lego stand-in
GEOMETRY_STEPS = 2000


@pytest.fixture(scope="module")
def lego_trained():
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=7))
    cfg = get_cfg()
    for split in ("train", "test"):
        cfg.dataset[split].n_images = 40
        cfg.dataset[split].H = cfg.dataset[split].W = 200
    cfg.dataset.val = None
    r = Runner()
    r.train(GEOMETRY_STEPS)
    torch.cuda.synchronize()
    return r


# |depth - t_hit| over the opaque pixels, measured on an NVIDIA H100 80GB HBM3 (700 W power limit): median 0.0079, 95th percentile
# 0.0331 NeRF units (two finest occupancy cells are 0.0473).  The bounds leave a margin of about 2.5x and 3x.
MEDIAN_BOUND, P95_BOUND = 0.02, 0.1


def test_depth_of_the_trained_lego_stand_in_matches_the_analytic_hit(lego_trained):
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg
    r = lego_trained
    ds = build_from_cfg(r.cfg.dataset.test, DATASETS)
    assert ds.n_images == 4 and ds.mode == "test"
    errs = []
    W, H = ds.resolution
    for i in range(ds.n_images):
        o, d = ds.generate_rays_total_test(i)
        rgba, t_hit = ds.shade(o, d, return_t=True)
        img, alpha, _, _, depth = r._render_frame(o, d, W, H, 1e-4, depth_scale=float(ds.scale))
        mask = (rgba[:, 3] == 1) & (alpha.reshape(-1) > 0.99)
        assert mask.sum() > 0.1 * H * W
        errs.append((depth.reshape(-1)[mask] - t_hit[mask] / ds.scale).abs().cpu().numpy())
    e = np.concatenate(errs)
    med, p95 = float(np.median(e)), float(np.percentile(e, 95))
    print(f"lego stand-in after {GEOMETRY_STEPS} steps, {e.size} opaque pixels of {ds.n_images} held-out views: |depth - t_hit| median "
          f"{med:.4f}, p95 {p95:.4f} NeRF units (two finest occupancy cells: {2 / 128 / ds.scale:.4f})")
    assert med <= MEDIAN_BOUND and p95 <= P95_BOUND, (med, p95)


def test_spiral_path_renders_the_trained_llff_stand_in(tmp_path_factory):
    from test_llff_gpu import _llff_runner
    from jnerf_b200.utils.camera_path import path_spiral
    root = str(tmp_path_factory.mktemp("llff_spiral"))
    r = _llff_runner(os.path.join(root, "fern"), seed=13, log_dir=os.path.join(root, "logs"))
    r.train(steps=600)
    ds = r.dataset["train"]
    path = path_spiral(ds.poses, ds.bounds, n_frames=8)
    near, far = r.depth_range(path)
    assert 0 < near < far and (near, far) == (float(ds.bounds.min()), float(ds.bounds.max()))
    for pose in path:
        img, depth, alpha = r.render_depth_with_pose(pose)
        assert img.shape == (ds.H, ds.W, 3) and depth.shape == (ds.H, ds.W)
        assert torch.isfinite(img).all() and torch.isfinite(depth).all()
        assert float((alpha > 0.5).float().mean()) > 0.9, float((alpha > 0.5).float().mean())
        covered = depth[alpha[..., 0] > 0.5]
        assert float(covered.median()) > 0.5 * near
    cv2 = pytest.importorskip("cv2")
    out = r.render(save_path=str(tmp_path_factory.mktemp("video") / "spiral.mp4"), depth=True, poses=path)
    cap = cv2.VideoCapture(out[:-4] + "_depth.mp4")
    k = 0
    while cap.read()[0]:
        k += 1
    cap.release()
    assert k == 8
