"""The whole-frame renderer on the H100, on lego and fox stand-ins trained for a few hundred steps (a non-trivial occupancy grid):
exact per-ray sample counts against ngp_march under the same jitter layout (const_dt, and cone stepping at aabb_scale 4), the image and
RNG of render_img_nosync at min_transmittance 0, the early-stopping bound, bit-identical results for any round capacity and from run to
run, and the edge cases (rays that miss the box, partial tiles, a single ray, rays that reach the step cap)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _runner(kind):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    if kind == "lego":
        update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=3))
        cfg = get_cfg()
        cfg.dataset.train.n_images = 16
        cfg.dataset.train.H = cfg.dataset.train.W = 160
        cfg.dataset.val = None
    else:
        update_cfg(**fox_cfg(fp16=True, synthetic=True, seed=3))
        cfg = get_cfg()
        cfg.dataset.train.n_images = 12
        cfg.dataset.train.H, cfg.dataset.train.W = 192, 108
    r = Runner()
    for _ in range(300):
        r.train_step()
    torch.cuda.synchronize()
    return r


@pytest.fixture(scope="module")
def runners():
    return {}


@pytest.fixture(params=["lego", "fox"])
def runner(request, runners):
    if request.param not in runners:
        runners[request.param] = _runner(request.param)
    return runners[request.param]


def render(r, o, d, eps, rng, capacity=None, bitfield=None, tile=None):
    from jnerf_b200 import ops
    s, m = r.sampler, r.model
    k = {} if capacity is None else {"capacity": capacity}
    return ops.render_rays(o.contiguous(), d.contiguous(), s.density_grid_bitfield if bitfield is None else bitfield, s.aabb_range,
                           s.cone_angle_constant, s.near_distance, s.NERF_CASCADES, s.const_dt, rng, m.pos_encoder.m_grid, m.pos_encoder.levels,
                           m.density_mlp.con_weights, m.rgb_mlp.con_weights, tile or r.cfg.n_rays_per_batch, min_transmittance=eps, **k)


def march_counts(r, o, d, rng, bitfield=None, tile=None):
    """Per-ray sample counts of ngp_march, one call per tile with one rng.advance() between tiles (render_img_nosync's layout)."""
    from jnerf_b200 import ops
    s = r.sampler
    tile = tile or r.cfg.n_rays_per_batch
    st, out = rng.copy(), []
    for p in range(0, o.shape[0], tile):
        _, _, numsteps, _ = ops.march(o[p:p + tile].contiguous(), d[p:p + tile].contiguous(),
                                      s.density_grid_bitfield if bitfield is None else bitfield, s.aabb_range, tile * 1024,
                                      s.cone_angle_constant, s.near_distance, s.NERF_CASCADES, s.const_dt, st)
        ops.pcg32_advance(st)
        out.append(numsteps[:, 0].cpu())
    return torch.cat(out)


def frame(r, img_id=0):
    return r.dataset["train"].generate_rays_total_test(img_id)


def test_sample_counts_equal_the_march(runner):
    r = runner
    o, d = frame(r, 1)
    rng = r.sampler.rng.copy()
    rgb, alpha, n, rounds = render(r, o, d, 0.0, rng)
    want = march_counts(r, o, d, rng)
    assert torch.equal(n.cpu(), want)
    assert want.sum() > 1000 and rounds >= 1
    assert r.sampler.const_dt == (r.cfg.exp_name == "lego")


def test_matches_render_img_nosync_at_eps_0(runner):
    r = runner
    s = r.sampler
    rng0 = s.rng.copy()
    img_ref, _ = r.render_img_nosync("train", 2)
    rng_ref = s.rng.copy()
    s.rng[:] = rng0
    o, d = frame(r, 2)
    rgb, alpha, n, _ = r.render_rays(o, d, min_transmittance=0.0)
    assert np.array_equal(s.rng, rng_ref)
    img = rgb + torch.tensor(r.background_color, dtype=torch.float32, device="cuda") * (1 - alpha)
    assert (img.reshape(img_ref.shape) - img_ref).abs().max().item() <= 1e-5


def test_early_stopping_bound(runner):
    r = runner
    o, d = frame(r, 3)
    rng = r.sampler.rng.copy()
    rgb0, a0, n0, _ = render(r, o, d, 0.0, rng)
    eps = 1e-4
    rgb1, a1, n1, _ = render(r, o, d, eps, rng)
    assert (n1 <= n0).all()
    for bg in ([0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [0.3, -0.5, 0.9]):
        b = torch.tensor(bg, device="cuda")
        diff = ((rgb1 + b * (1 - a1)) - (rgb0 + b * (1 - a0))).abs().max().item()
        assert diff <= eps * (1 + max(abs(x) for x in bg)) + 1e-5, (bg, diff)
    if r.cfg.exp_name == "lego":
        assert n1.float().mean() < n0.float().mean()


def test_bit_identical_for_any_capacity_and_run(runner):
    r = runner
    o, d = frame(r, 4)
    rng = r.sampler.rng.copy()
    assert o.shape[0] > 1 << 12
    for eps in (0.0, 1e-4):
        # 2^12 rows hold fewer rows than there are rays: one sample a ray, and only the first 2^12 alive rays march in a round
        a = render(r, o, d, eps, rng, capacity=1 << 12)
        b = render(r, o, d, eps, rng, capacity=1 << 16)
        c = render(r, o, d, eps, rng, capacity=1 << 21)
        e = render(r, o, d, eps, rng, capacity=1 << 21)
        assert a[3] > b[3] > c[3]                                      # smaller capacities take more rounds
        for x, y, z, w in zip(a[:3], b[:3], c[:3], e[:3]):
            assert torch.equal(x, y) and torch.equal(y, z) and torch.equal(z, w)


def test_rays_whose_t_stops_growing_end_at_the_step_guard(runner):
    """Rays the reference's loop would march for ever: an origin far from the box (t + dt == t once t passes ~16 k with const_dt), a
    direction of tiny length (its skip target lies far beyond where t stops growing) and a zero direction.  Both marches stop them
    after MARCH_STEP_GUARD steps of the t sequence; the sample counts agree, with the trained grid and with every cell occupied."""
    r = runner
    lo, hi = r.sampler.aabb_range
    mid = 0.5 * (lo + hi)
    o = torch.tensor([[lo - 2.0e4, mid, mid], [mid, mid, mid], [mid, mid, mid], [mid + 0.1, mid - 0.2, mid]], device="cuda")
    d = torch.tensor([[1.0, 0.0, 0.0], [1e-7, 0.0, 0.0], [0.0, 0.0, 0.0], [3e-7, 2e-7, -1e-7]], device="cuda")
    rng = r.sampler.rng.copy()
    full = torch.full_like(r.sampler.density_grid_bitfield, 255)
    for bits in (None, full):
        for eps in (0.0, 1e-4):
            rgb, alpha, n, _ = render(r, o, d, eps, rng, bitfield=bits)
            assert torch.isfinite(rgb).all() and torch.isfinite(alpha).all()
            if eps == 0.0:
                assert torch.equal(n.cpu(), march_counts(r, o, d, rng, bitfield=bits))
    assert (n.cpu()[1:3] > 0).all()                                    # every cell occupied: the stuck rays still composite samples
    from jnerf_b200 import lib
    torch.cuda.synchronize()
    assert lib.load().ngp_debug_timeout_flag() == 0


def test_edge_cases(runners):
    if "lego" not in runners:
        runners["lego"] = _runner("lego")
    r = runners["lego"]
    from jnerf_b200 import lib
    o, d = frame(r, 5)
    rng = r.sampler.rng.copy()
    # rays that miss the box: outside it and pointing away
    miss_o = torch.tensor([[3.0, 3.0, 3.0]] * 7, device="cuda")
    miss_d = torch.nn.functional.normalize(torch.tensor([[1.0, 0.7, 0.2]] * 7, device="cuda"), dim=1)
    rgb, alpha, n, _ = render(r, miss_o, miss_d, 1e-4, rng)
    assert (n == 0).all() and (rgb == 0).all() and (alpha == 0).all()
    # R not a multiple of the tile, a partial tile of another tile size, and R = 1
    for R, tile in ((1000, None), (5003, 1024), (1, None)):
        oo, dd = o[1000:1000 + R], d[1000:1000 + R]
        rgb, alpha, n, _ = render(r, oo, dd, 0.0, rng, tile=tile)
        assert torch.equal(n.cpu(), march_counts(r, oo, dd, rng, tile=tile))
    # rays that reach the step cap: every cell occupied, rays along the diagonal of the unit cube (2048 steps of the constant dt)
    full = torch.full_like(r.sampler.density_grid_bitfield, 255)
    cap_o = torch.tensor([[-0.5, -0.5, -0.5], [1.5, -0.5, -0.5]], device="cuda")
    cap_d = torch.nn.functional.normalize(torch.tensor([[1.0, 1.0, 1.0], [-1.0, 1.0, 1.0]], device="cuda"), dim=1)
    oo, dd = torch.cat([cap_o, o[:500]]), torch.cat([cap_d, d[:500]])
    rgb, alpha, n, _ = render(r, oo, dd, 0.0, rng, bitfield=full, capacity=1 << 16)
    want = march_counts(r, oo, dd, rng, bitfield=full)
    assert torch.equal(n.cpu(), want) and (n[:2] == 1024).all()
    torch.cuda.synchronize()
    assert lib.load().ngp_debug_timeout_flag() == 0
