"""The single-GPU training tail: ngp_network_bwd_fx into caller-owned scratch + one ngp_train_sweep must give the parameters and
optimizer state that ngp_network_bwd + three ngp_adam_ema sweeps give, bit for bit, and leave the scratch zeroed; a Runner that uses
it trains identically pipelined and sequential."""
import pytest
import torch

pytestmark = pytest.mark.gpu

HYPER = dict(beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95)
LR = 1e-2
# ngp_network_bwd keeps its scratch per stream and sizes it when it first sees a level table's address: a later table at a freed
# table's address would find scratch sized for the old one (include/ngp_b200.h).  The tables of this module stay alive.
_TABLES = []


def _inputs(aabb, n_max, n_live, seed):
    from jnerf_b200 import ops
    lv = ops.HashLevels(aabb, log2_hashmap_size=19)
    _TABLES.append(lv)
    g = torch.Generator(device="cuda").manual_seed(seed)
    coords = torch.rand((n_max, 7), device="cuda", generator=g)
    grid = ((torch.rand(lv.n_params, device="cuda", generator=g) - 0.5) * 2e-2).half()
    wd = ((torch.rand(3072, device="cuda", generator=g) - 0.5) * 0.5).half()
    wr = ((torch.rand(7168, device="cuda", generator=g) - 0.5) * 0.5).half()
    n_dev = None if n_live is None else torch.tensor([n_live], dtype=torch.int32, device="cuda")
    _, enc = ops.network_fwd(coords, grid, lv, wd, wr, n_dev=n_dev)
    dout = (torch.randn((n_max, 4), device="cuda", generator=g) * 0.05).half()
    return lv, coords, enc, dout, n_dev, [grid, wd, wr]


def _state(params):
    return [(torch.zeros(p.numel(), device="cuda"), torch.zeros(p.numel(), device="cuda"), p.float().clone()) for p in params]


@pytest.mark.parametrize("aabb,n_max,n_live", [(1, 1 << 18, None), (4, 1 << 18, None), (1, 70001, None), (4, 70001, 41234)],
                         ids=["lego-2^18", "fox-2^18", "lego-70001", "fox-70001-live41234"])
def test_bwd_fx_plus_sweep_equals_bwd_plus_three_sweeps(aabb, n_max, n_live):
    from jnerf_b200 import ops
    lv, coords, enc, dout, n_dev, p0 = _inputs(aabb, n_max, n_live, seed=5 + n_max + aabb)
    pa, pb = [p.clone() for p in p0], [p.clone() for p in p0]
    sa, sb = _state(pa), _state(pb)
    gg = torch.zeros(lv.n_params, dtype=torch.float16, device="cuda")
    dwd, dwr = torch.zeros(3072, device="cuda"), torch.zeros(7168, device="cuda")
    fx, part = ops.network_bwd_scratch(lv)
    for step in (1, 2):                                      # the second backward runs on the updated weights, into the cleared scratch
        ops.network_bwd(coords, enc, lv, pa[1], pa[2], dout, gg, dwd, dwr, n_dev=n_dev)
        for p, gr, (m, v, ms) in zip(pa, (gg, dwd, dwr), sa):
            ops.adam_ema(p, gr, m, v, ms, LR, step, **HYPER, grad_scale=1.0, zero_grad=True)
        ops.network_bwd_fx(coords, enc, lv, pb[1], pb[2], dout, fx, part, n_dev=n_dev)
        ops.train_sweep(pb[0], sb[0], fx, part, n_max, pb[1], sb[1], pb[2], sb[2], LR, step, **HYPER)
        torch.cuda.synchronize()
        assert int(torch.count_nonzero(fx)) == 0, "the sweep must leave the scratch zeroed"
        for k, name in enumerate(("table", "density weights", "colour weights")):
            assert torch.equal(pa[k].view(torch.int16), pb[k].view(torch.int16)), (step, name)
            for t, (x, y) in zip(("m", "v", "master"), zip(sa[k], sb[k])):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (step, name, t)
    assert not torch.equal(pa[0], p0[0]) and not torch.equal(pa[2], p0[2])
    assert ops.lib.load().ngp_debug_timeout_flag() == 0


def test_bwd_fx_refuses_short_scratch():
    from jnerf_b200 import lib, ops
    lv, coords, enc, dout, _, (grid, wd, wr) = _inputs(1, 4096, None, seed=3)
    fx, part = ops.network_bwd_scratch(lv)
    with pytest.raises(lib.NgpError, match="16 bytes per table entry"):
        ops.network_bwd_fx(coords, enc, lv, wd, wr, dout, fx[:-2], part)
    with pytest.raises(lib.NgpError, match="weight-gradient slots"):
        ops.network_bwd_fx(coords, enc, lv, wd, wr, dout, fx, part[:-1])


def _train(monkeypatch, steps, **env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=29))
    cfg = get_cfg()
    cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W, cfg.dataset.val = 8, 160, 160, None
    r = Runner()
    assert r._fx is not None
    losses = [r.train_step().clone() for _ in range(steps)]
    torch.cuda.synchronize()
    return r, torch.stack([l.mean() for l in losses]), {k: v.detach().clone() for k, v in r.model.state_dict().items()}


def test_runner_pipelined_equals_sequential_bit_for_bit(monkeypatch):
    """64 steps = four occupancy-grid updates: the deterministic backward and sweep make the two step orders train identically."""
    ra, la, pa = _train(monkeypatch, 64, NGP_PIPELINE="1")
    assert ra._pipe is not None and ra._pipe["prefetched"] > 0
    rb, lb, pb = _train(monkeypatch, 64, NGP_PIPELINE="0")
    assert rb._pipe is None
    assert torch.equal(la, lb)
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k

