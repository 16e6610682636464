"""End-to-end checks of the plugin classes and the training driver on a GPU: the fused fast path equals the per-operator
autograd path (the way JNeRF's Runner wires the ops), training converges on the synthetic scene, checkpoints round-trip,
and data-parallel sharding on ONE device reproduces the single-rank gradients."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def make_runner(seed=1, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=seed, **over))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 8
    cfg.dataset.train.H = cfg.dataset.train.W = 160
    cfg.dataset.val = None
    return Runner()


def test_plugin_api_surface():
    r = make_runner()
    m, s = r.model, r.sampler
    # names / attributes the reference exposes (SURVEY.md 8b)
    assert m.pos_encoder.out_dim == 32 and m.dir_encoder.out_dim == 16 and m.pos_encoder.m_grid.numel() == 12196240
    assert m.density_mlp.con_weights.numel() == 3072 and m.rgb_mlp.con_weights.numel() == 7168
    assert s.n_rays_per_batch == 4096 and s.density_grid.numel() == 5 * 128 ** 3 and s.density_grid_bitfield.numel() == 5 * 128 ** 3 // 8
    pos = torch.rand(1000, 3, device="cuda")
    dirs = torch.rand(1000, 3, device="cuda")
    out = m(pos, dirs)
    assert out.shape == (1000, 4) and out.dtype == torch.float16
    assert m.density(pos).shape == (1000, 1)
    enc = m.pos_encoder(pos)
    assert enc.shape == (1000, 32) and enc.dtype == torch.float16
    # the fused network == the per-operator composition (ngp_network.py:77-84)
    ref = m.execute_(pos, dirs)
    assert (out.float() - ref.float()).abs().max() < 2e-2
    assert (m.density(pos).float() - ref[:, 3:].float()).abs().max() < 1e-2


def test_fused_step_equals_autograd_step():
    """Same batch, same parameters: the gradients of the fused fast path equal those torch autograd derives through the per-operator
    plugin classes (the way JNeRF wires the ops).  After one step Adam's first moment is exactly (1-beta1) * gradient."""
    ra = make_runner(seed=3)
    la = ra.train_step()
    rb = make_runner(seed=3)
    lb = rb.train_step_autograd()
    assert abs(float(la.mean()) - float(lb.detach().mean())) < 5e-3 * max(1.0, float(lb.detach().mean()))
    sa, sb = ra.optimizer._nested_optimizer.state, rb.optimizer._nested_optimizer.state
    for a, b, tol in zip(sa, sb, (5e-2, 3e-2, 3e-2)):          # hash grid (fp16 atomics), density MLP, colour MLP
        ga, gb = a.m / 0.1, b.m / 0.1
        scale = float(gb.abs().max())
        assert scale > 0
        assert float((ga - gb).abs().max()) <= tol * scale, (float((ga - gb).abs().max()), scale)
        assert float((ga - gb).abs().mean()) <= 2e-3 * scale
    # and a few more steps stay together in loss
    for _ in range(3):
        la, lb = ra.train_step(), rb.train_step_autograd()
    assert abs(float(la.mean()) - float(lb.detach().mean())) < 2e-2 * max(1.0, float(lb.detach().mean()))


def test_training_converges_and_renders():
    r = make_runner(seed=5)
    first = float(r.train_step().mean())
    for _ in range(299):
        loss = r.train_step()
    last = float(loss.mean())
    assert np.isfinite(last) and last < 0.5 * first, (first, last)
    assert int(r.sampler.density_grid_bitfield.count_nonzero()) > 0
    psnr = r.psnr("train", max_images=2)
    assert psnr > 18.0, psnr                                          # 300 steps on 8 small views
    from jnerf_b200 import ops
    assert ops.lib.load().ngp_debug_timeout_flag() == 0


def test_checkpoint_roundtrip(tmp_path):
    r = make_runner(seed=7)
    for _ in range(20):
        r.train_step()
    p = str(tmp_path / "ckpt.pt")
    r.save_ckpt(p)
    g0 = r.model.pos_encoder.m_grid.detach().clone()
    r2 = make_runner(seed=9)
    r2.load_ckpt(p)
    assert torch.equal(r2.model.pos_encoder.m_grid.detach(), g0)
    assert torch.equal(r2.sampler.density_grid_bitfield, r.sampler.density_grid_bitfield)
    assert r2.cfg.m_training_step == 20 and r2.optimizer._nested_optimizer.n_step == 20


def test_dp_shards_reproduce_single_rank_gradients():
    """Two data-parallel shards executed one after the other on one device: summed, 1/W-scaled gradients of the shards equal the
    single-rank gradients of the global batch (SURVEY.md 8e), and the shard samples are the global samples."""
    from jnerf_b200 import dp, ops
    r = make_runner(seed=11)
    for _ in range(32):
        r.train_step()                                                  # carve the occupancy grid first
    s, m = r.sampler, r.model
    ds = r.dataset["train"]
    R = 96                                                              # small enough that the sample capacity never truncates
    pix = ds.next_pixels(2 * R)
    bg = torch.rand((2 * R, 3), device="cuda")
    mean = s.density_grid_mean

    def grads(pix_, bg_, offset):
        ids, o, d = ds.rays_for(pix_)
        rgba = ds.rgba_for(pix_)
        target = (rgba[:, :3] * rgba[:, 3:] + bg_ * (1 - rgba[:, 3:])).contiguous()
        rng = ops.pcg32_advance(s.rng.copy(), offset * 8) if offset else s.rng
        coords, _, ns, cnt = ops.march(o, d, s.density_grid_bitfield, s.aabb_range, s.max_samples, s.cone_angle_constant, s.near_distance,
                                       s.NERF_CASCADES, s.const_dt, rng)
        _, ns_c, cnt_c = ops.compact(coords, ns, s.target_batch_size, alias=True)
        n = int(cnt_c[0])
        c = coords[:s.target_batch_size]
        out, enc = ops.network_fwd(c, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, n_dev=cnt_c[0:1])
        _, _, dnet = ops.composite_loss_bwd(out, c, ns, ns_c, bg_.contiguous(), target, mean)
        gg = torch.zeros_like(m.pos_encoder.m_grid.data)
        dwd, dwr = torch.zeros(3072, device="cuda"), torch.zeros(7168, device="cuda")
        ops.network_bwd(c, enc, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, dnet, gg, dwd, dwr, n_dev=cnt_c[0:1])
        return gg.float(), dwr, ns[:, 0].clone(), n

    g_full, w_full, ns_full, n_full = grads(pix, bg, 0)
    parts = [grads(pix[k * R:(k + 1) * R], bg[k * R:(k + 1) * R], dp.shard_range(R, k)[0]) for k in range(2)]
    assert torch.equal(torch.cat([parts[0][2], parts[1][2]]), ns_full)            # identical samples per ray
    assert parts[0][3] + parts[1][3] == n_full and n_full < s.target_batch_size
    g_sum = (parts[0][0] + parts[1][0]) * 0.5                                     # all-reduce(sum) then x 1/W
    w_sum = (parts[0][1] + parts[1][1]) * 0.5
    assert (w_sum - w_full).abs().max() <= 2e-2 * w_full.abs().max()
    assert (g_sum - g_full).abs().max() <= 5e-2 * g_full.abs().max() and (g_sum - g_full).abs().mean() <= 2e-3 * g_full.abs().max()


def _same_sampling(cnt_a, ns_a, cnt_b, ns_b):
    """Two runs of the same seeds after occupancy-grid rebuilds: not bit for bit (both grids come from networks whose gradients were
    summed by atomics in a different order, and the adaptive ray batch moves in multiples of 128 rays), but the same sampling density:
    fraction of rays that hit occupied space and samples per such ray within 3 %."""
    hit_a, hit_b = int(cnt_a[1]) / ns_a.shape[0], int(cnt_b[1]) / ns_b.shape[0]
    per_a, per_b = int(cnt_a[0]) / max(int(cnt_a[1]), 1), int(cnt_b[0]) / max(int(cnt_b[1]), 1)
    assert abs(ns_a.shape[0] - ns_b.shape[0]) <= 256, (ns_a.shape, ns_b.shape)
    assert abs(hit_a - hit_b) <= 0.03 * hit_b and abs(per_a - per_b) <= 0.03 * per_b, (hit_a, hit_b, per_a, per_b)


def test_pipelined_steps_match_sequential_steps(monkeypatch):
    """The software pipeline over steps (march of step i+1 on a second stream under step i's backward / optimizer sweep) against the
    strictly sequential step with the same seeds: the same pixels, the same rays and samples until the first occupancy-grid rebuild
    (bit for bit: the march reads nothing the network kernels write), losses equal up to the order of the gradient atomics, and the
    same training progress afterwards.  Exact equality of the two orders is tests/test_runner_cpu.py's (deterministic oracle)."""
    import numpy as np
    from jnerf_b200 import ops
    runs = {}
    for pipe in ("1", "0"):
        monkeypatch.setenv("NGP_PIPELINE", pipe)
        r = make_runner(seed=23)
        assert (r._pipe is not None) == (pipe == "1")
        losses, marks = [], []
        for k in range(120):
            losses.append(float(r.train_step().mean()))
            if k in (7, 40):
                marks.append((r.sampler._counters_compacted.clone(), r.sampler._rays_numsteps.clone()))
        runs[pipe] = dict(losses=np.array(losses), marks=marks, n_step=r.optimizer._nested_optimizer.n_step, rays=r.sampler.n_rays_per_batch,
                          prefetched=r._pipe["prefetched"] if r._pipe is not None else 0)
        img, tar = r.render_img_nosync("train", 0)
        runs[pipe]["psnr"] = float(-10.0 * torch.log10(((img - tar) ** 2).mean()))
        assert ops.lib.load().ngp_debug_timeout_flag() == 0
    a, b = runs["1"], runs["0"]
    assert a["prefetched"] == 120 - 7 and a["n_step"] == b["n_step"] == 120       # all but the fronts of steps 16, 32 .. 112 (grid update first)
    (cnt_a, ns_a), (cnt_b, ns_b) = a["marks"][0], b["marks"][0]
    assert torch.equal(cnt_a, cnt_b) and torch.equal(ns_a, ns_b)                  # step 7: same occupancy grid, same jitter -> same samples
    (cnt_a, ns_a), (cnt_b, ns_b) = a["marks"][1], b["marks"][1]
    _same_sampling(cnt_a, ns_a, cnt_b, ns_b)
    la, lb = a["losses"], b["losses"]
    assert np.all(np.isfinite(la)) and np.abs(la[:16] - lb[:16]).max() <= 2e-3 * np.abs(lb[:16]).max()
    assert np.abs(la[:41] - lb[:41]).max() <= 5e-2 * np.abs(lb).max() and abs(la[-8:].mean() - lb[-8:].mean()) <= 0.1 * lb[-8:].mean()
    assert abs(a["psnr"] - b["psnr"]) < 0.5 and a["psnr"] > 18.0, (a["psnr"], b["psnr"])
