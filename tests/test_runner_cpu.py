"""Host logic of the plugin classes and the Runner, exercised without a GPU: the operator layer is swapped for the oracle and
torch's "cuda" for "cpu" (tests/cpu_backend.py).  What is under test is everything AROUND the kernels -- the order of the C-ABI
calls in a training step (runner/runner.py:62-84 of the reference), buffer aliasing, gradient zeroing, the adaptive ray batch
(density_grid_sampler.py:266-271), optimizer / EMA step order, both checkpoint formats, the two tiled renderers, the fox
configuration -- not the kernels, which `-m gpu` checks against the same oracle."""
import numpy as np
import pytest
import torch

import cpu_backend
import oracle_lib as ol


def make_runner(monkeypatch, cfg_fn="lego_cfg", images=4, H=24, W=24, rays=64, target=32768, seed=1, start_step=1, pipeline=False, **over):
    fake = cpu_backend.install(monkeypatch)
    # pipeline=False: the strictly sequential step (one step's calls, then the next's); the software pipeline over steps has its own tests
    monkeypatch.setenv("NGP_PIPELINE", "1" if pipeline else "0")
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**getattr(R, cfg_fn)(fp16=True, synthetic=True, seed=seed, n_rays_per_batch=rays, target_batch_size=target, **over))
    cfg = get_cfg()
    cfg.dataset.train.n_images = images
    cfg.dataset.train.H, cfg.dataset.train.W = H, W
    cfg.dataset.val = None
    r = R.Runner()
    # skip the first occupancy-grid update (2 M density evaluations at step 0: minutes with the scalar oracle); it has its own test
    bits, _ = ol.sphere_bitfield(0.35, cascades=r.sampler.NERF_CASCADES)
    r.sampler.density_grid_bitfield.copy_(torch.from_numpy(bits[:r.sampler.density_grid_bitfield.numel()]))
    cfg.m_training_step = start_step
    return r, fake


STEP_OPS = ["prepare_batch", "march", "compact", "network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema", "adam_ema", "adam_ema"]


def test_sequential_step_call_sequence_and_bookkeeping(monkeypatch):
    r, fake = make_runner(monkeypatch)
    m, s = r.model, r.sampler
    assert r.fast and m.pos_encoder.m_grid.numel() == 12196240 and s.max_samples == 64 * 1024
    g0 = m.pos_encoder.m_grid.detach().clone()
    w0 = m.rgb_mlp.con_weights.detach().clone()
    rng0 = s.rng.copy()
    fake.calls.clear()
    loss = r.train_step()
    assert fake.calls == STEP_OPS                                   # one C-ABI call per stage, in the reference's order
    assert torch.isfinite(loss).all() and loss.shape == (64,)
    assert r.cfg.m_training_step == 2 and r.optimizer._nested_optimizer.n_step == 1 and r.ema_optimizer.steps == 1 and r.optimizer.steps == 1
    assert not torch.equal(m.pos_encoder.m_grid.detach(), g0) and not torch.equal(m.rgb_mlp.con_weights.detach(), w0)
    assert not r.grid_grad.any() and not r.dwd.any() and not r.dwr.any()          # the optimizer sweep zeroes the gradients
    assert np.array_equal(s.rng, ol.pcg32_advance(rng0.copy()))                   # one rng.advance() per march (ray_sampler.py:61)
    n_samples = int(s.n_samples_dev.item())
    assert 0 < n_samples <= s.target_batch_size and int(s.measured_batch_size.item()) == n_samples   # 64 rays fit the sample budget
    # Adam's first moment after one step is (1 - beta1) * gradient: non-zero exactly where the table was touched
    st = r.optimizer._nested_optimizer.state[0]
    assert 0 < int((st.m != 0).sum()) < st.m.numel()
    # steps 2..15: the 16th iteration of the window adapts the ray batch to the measured sample count (density_grid_sampler.py:266-271)
    first = float(loss.mean())
    fake.calls.clear()
    loss = r.train_step()
    assert fake.calls == STEP_OPS
    for _ in range(12):
        loss = r.train_step()
    assert r.cfg.m_training_step == 15 and s.n_rays_per_batch == 64
    measured = int(s.measured_batch_size.item())
    loss = r.train_step()                                                          # i = 15
    expect = int(64 * s.target_batch_size / max((measured + int(s.n_samples_dev.item())) / 16, 1))
    expect = min((expect + 127) // 128 * 128, s.target_batch_size)
    assert s.n_rays_per_batch == expect and r.dataset["train"].batch_size == expect and int(s.measured_batch_size.item()) == 0
    assert np.isfinite(float(loss.mean())) and np.isfinite(first)


def test_fused_step_equals_per_operator_autograd_step(monkeypatch):
    """Runner.train_step (fused C-ABI calls) and Runner.train_step_autograd (the per-operator plugin classes under autograd, the way
    JNeRF's Runner wires them) produce the same gradients: Adam's first moment after one step is (1 - beta1) * gradient."""
    ra, _ = make_runner(monkeypatch, seed=3)
    la = ra.train_step()
    ma = [st.m.clone() for st in ra.optimizer._nested_optimizer.state]
    rb, _ = make_runner(monkeypatch, seed=3)
    lb = rb.train_step_autograd()
    mb = [st.m for st in rb.optimizer._nested_optimizer.state]
    assert abs(float(la.mean()) - float(lb.detach().mean())) < 2e-3 * max(1.0, float(lb.detach().mean()))
    for a, b, tol in zip(ma, mb, (3e-2, 2e-2, 2e-2)):
        scale = float(b.abs().max())
        assert scale > 0 and float((a - b).abs().max()) <= tol * scale, (float((a - b).abs().max()), scale)


def test_checkpoints_native_and_reference_format(monkeypatch, tmp_path):
    r, _ = make_runner(monkeypatch, seed=5)
    for _ in range(4):
        r.train_step()
    for name in ("ckpt.pt", "params.pkl"):
        p = str(tmp_path / name)
        r.cfg.m_training_step = 5                                 # cfg is a process-wide singleton (as in the reference): r2 below shares it
        r.save_ckpt(p)
        r2, _ = make_runner(monkeypatch, seed=6)
        r2.load_ckpt(p)
        assert torch.equal(r2.model.pos_encoder.m_grid.detach(), r.model.pos_encoder.m_grid.detach())
        assert torch.equal(r2.model.density_mlp.con_weights.detach(), r.model.density_mlp.con_weights.detach())
        assert torch.equal(r2.sampler.density_grid_bitfield, r.sampler.density_grid_bitfield)
        assert r2.cfg.m_training_step == 5 and r2.start == 5 and r2.optimizer._nested_optimizer.n_step == 4 and r2.ema_optimizer.steps == 4
        assert r2.optimizer.steps == 4 and np.array_equal(r2.sampler.rng, r.sampler.rng)
        a, b = r.optimizer._nested_optimizer.state[2], r2.optimizer._nested_optimizer.state[2]
        if name.endswith(".pt"):
            assert torch.equal(a.m, b.m) and torch.equal(a.v, b.v) and torch.equal(a.master, b.master)
        else:
            # a .pkl written here round-trips losslessly (fp32 state under extra keys the reference ignores) ...
            assert torch.equal(a.m, b.m) and torch.equal(a.v, b.v) and torch.equal(a.master, b.master)
            from jnerf_b200.utils import ckpt_compat as cc
            ref = cc.read_reference_ckpt(p)                       # ... and has the fields the reference's load_ckpt indexes (runner.py:133-151),
            pg = ref["nested_optimizer"]["defaults"]["param_groups"][0]      # in the parameter dtype, as Jittor keeps them
            assert ref["global_step"] == 5 and len(pg["values"]) == 3 and pg["values"][0].dtype == np.float16 and pg["m"][0].dtype == np.float16
            assert ref["ema_optimizer"]["defaults"]["steps"] == 4
        assert torch.isfinite(r2.train_step()).all()


def test_both_tiled_renderers_agree(monkeypatch):
    r, fake = make_runner(monkeypatch, seed=7)
    for _ in range(3):
        r.train_step()
    rng0 = r.sampler.rng.copy()
    fake.calls.clear()
    img_a, tar_a = r.render_img("train", 1)
    n_tiles = (24 * 24 + 63) // 64
    assert fake.calls.count("march") == n_tiles and fake.calls.count("composite_infer") == n_tiles
    rng1 = r.sampler.rng.copy()
    r.sampler.rng = rng0.copy()
    img_b, tar_b = r.render_img_nosync("train", 1)
    assert np.array_equal(r.sampler.rng, rng1)
    assert torch.equal(tar_a, tar_b) and torch.equal(img_a, img_b)
    assert img_a.shape == (24, 24, 3) and float(img_a.std()) > 0
    assert np.isfinite(r.psnr("train", max_images=1))


def test_fox_configuration_runs(monkeypatch):
    r, fake = make_runner(monkeypatch, cfg_fn="fox_cfg", images=3, H=32, W=18, seed=2)
    s = r.sampler
    assert r.dataset["train"].aabb_scale == 4 and s.aabb_range == (-1.5, 2.5) and s.max_cascade == 2 and s.const_dt is False
    assert r.model.pos_encoder.m_grid.numel() == 2 * 6537456
    l0 = float(r.train_step().mean())
    for _ in range(5):
        loss = r.train_step()
    assert np.isfinite(float(loss.mean())) and float(loss.mean()) < l0
    assert fake.calls.count("march") == 6
    # occupancy-grid update over the three cascades an aabb_scale of 4 uses (max_cascade + 1, density_grid_sampler.py:233)
    r.cfg.m_training_step = 0
    s.update_density_grid_nerf(0.95, 30000, 0)
    G3 = 128 ** 3 // 8
    bits = s.density_grid_bitfield
    assert int(bits[:G3].count_nonzero()) > 0 and int(bits[G3:3 * G3].count_nonzero()) > 0 and float(s.density_grid_mean.item()) > 0


def test_occupancy_grid_update_glue(monkeypatch):
    """update_density_grid_nerf (density_grid_sampler.py:204-250) at step 0 with a reduced sample count: mark_untrained, sample
    generation with the shared RNG stream, density evaluation, splat, EMA, bitfield -- in that order, RNG advanced once per
    non-empty generate call (SURVEY H5)."""
    r, fake = make_runner(monkeypatch, start_step=0)
    s = r.sampler
    rng0 = s.rng.copy()
    fake.calls.clear()
    s.update_density_grid_nerf(0.95, 20000, 0)
    assert fake.calls == ["grid_mark_untrained", "grid_generate_samples", "density_fwd", "grid_splat", "grid_ema", "grid_update_bitfield"]
    assert np.array_equal(s.rng, ol.pcg32_advance(rng0.copy())) and int(s.density_grid_ema_step.item()) == 1
    assert int(s.density_grid_bitfield.count_nonzero()) > 0 and float(s.density_grid_mean.item()) > 0
    r.cfg.m_training_step = 300
    fake.calls.clear()
    s.update_density_grid_nerf(0.95, 5000, 5000)
    assert fake.calls == ["grid_generate_samples", "grid_generate_samples", "density_fwd", "grid_splat", "grid_ema", "grid_update_bitfield"]
    assert np.array_equal(s.rng, ol.pcg32_advance(ol.pcg32_advance(ol.pcg32_advance(rng0.copy()))))


# ------------------------------------------------------------------------------------------------ data parallel (gloo, 2 ranks)
def _dp_worker(rank, world, port, tmp, ret, pipeline=False, start_step=1, steps=3):
    import os
    import sys
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), NGP_DP_EXCHANGE="nccl")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    torch.set_num_threads(1)
    mp_ = pytest.MonkeyPatch()
    try:
        fake = cpu_backend.install(mp_)
        mp_.setenv("NGP_PIPELINE", "1" if pipeline else "0")
        from jnerf_b200 import plugin  # noqa: F401
        from jnerf_b200 import runner as R
        from jnerf_b200.utils.config import get_cfg, update_cfg
        get_cfg().clear()
        update_cfg(**R.lego_cfg(fp16=True, synthetic=True, seed=1, n_rays_per_batch=32, target_batch_size=16384))
        cfg = get_cfg()
        cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W = 4, 24, 24
        cfg.dataset.val = None
        r = R.Runner(rank=rank, world_size=world, process_group=dist.group.WORLD)
        bits, _ = ol.sphere_bitfield(0.35)
        r.sampler.density_grid_bitfield.copy_(torch.from_numpy(bits))
        cfg.m_training_step = start_step
        r.sampler.update_density_grid = lambda: None               # 2 M density evaluations in the scalar oracle; it has its own test
        assert r.dp_mode == "nccl" and r._hi - r._lo == r._table.numel() // world
        losses, rays = [], []
        for _ in range(steps):
            rays.append(r.sampler.n_rays_per_batch)
            losses.append(float(r.train_step().mean()))
        rays.append(r.sampler.n_rays_per_batch)
        r._table_ready()
        assert (r._pipe is not None) == pipeline
        g = r.model.pos_encoder.m_grid.detach().float()
        st = r.optimizer._nested_optimizer.state[0]
        r.save_ckpt(os.path.join(tmp, "dp.pt"))                                  # every rank calls; rank 0 writes the gathered state
        ret[rank] = dict(losses=losses, table_sum=float(g.double().sum()), table_head=g[:4096].clone().numpy(), w=r.model.rgb_mlp.con_weights.detach().float().numpy(),
                         slice_len=int(st.m.numel()), calls=list(fake.calls[-9:]), n_samples=int(r.sampler.n_samples_dev.item()), rays=rays)
    finally:
        mp_.undo()
        dist.destroy_process_group()


def test_two_rank_runner_sharded_optimizer_keeps_replicas_identical(tmp_path):
    """Runner with world_size 2 over gloo (NCCL code path of runner._optimizer_step: reduce-scatter, Adam+EMA on this rank's slice of
    the padded table, all-gather awaited after the next march): both ranks hold the same table and MLP weights after every step although
    each optimises only half of the table; each rank marches its own shard of the global ray batch; the checkpoint gathers the slices."""
    import os
    import torch.multiprocessing as mp
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_dp_worker, args=(world, 29711 + os.getpid() % 1000, str(tmp_path), ret), nprocs=world, join=True)
    a, b = ret[0], ret[1]
    assert a["table_sum"] == b["table_sum"] and np.array_equal(a["table_head"], b["table_head"]) and np.array_equal(a["w"], b["w"])
    assert a["slice_len"] == b["slice_len"] == (12196240 + 511) // 512 * 512 // 2
    assert a["n_samples"] != b["n_samples"] or a["losses"] != b["losses"]        # different shards of the batch
    assert all(np.isfinite(a["losses"])) and all(np.isfinite(b["losses"]))
    assert a["calls"] == ["prepare_batch", "march", "compact", "network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema", "adam_ema", "adam_ema"]
    ck = torch.load(str(tmp_path / "dp.pt"), map_location="cpu", weights_only=False)
    assert ck["nested_optimizer"]["m"][0].numel() == 12196240 and ck["global_step"] == 4
    # the same two ranks with the software pipeline over steps (march of step i+1 enqueued under step i, the exchange of step i-1
    # awaited right before the network forward): the same losses and the same table, to the last bit
    ret2 = mp.Manager().dict()
    mp.spawn(_dp_worker, args=(world, 29713 + os.getpid() % 1000, str(tmp_path), ret2, True), nprocs=world, join=True)
    for k in (0, 1):
        assert ret2[k]["losses"] == ret[k]["losses"] and ret2[k]["table_sum"] == ret[k]["table_sum"] and np.array_equal(ret2[k]["w"], ret[k]["w"])
    assert ret2[0]["calls"][-3:] == ["prepare_batch", "march", "compact"]          # the prefetched front of the next step


def test_real_capture_through_the_runner(monkeypatch, tmp_path):
    """ngp_fox.py on the reduced real capture (tests/golden/fox_small, NerfDataset): a few training steps and a rendered tile."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_fox_small import materialise
    root = materialise(str(tmp_path / "fox"))
    fake = cpu_backend.install(monkeypatch)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**R.fox_cfg(fp16=True, synthetic=False, seed=1, n_rays_per_batch=48, target_batch_size=32768))
    cfg = get_cfg()
    cfg.dataset.train.root_dir = root
    cfg.dataset.test.root_dir = root
    r = R.Runner()
    ds = r.dataset["train"]
    assert type(ds).__name__ == "NerfDataset" and ds.n_images == 50 and ds.aabb_scale == 4 and r.sampler.aabb_range == (-1.5, 2.5)
    bits, _ = ol.sphere_bitfield(0.35)
    r.sampler.density_grid_bitfield.copy_(torch.from_numpy(bits))
    cfg.m_training_step = 1
    losses = [float(r.train_step().mean()) for _ in range(4)]
    assert all(np.isfinite(losses)) and fake.calls.count("prepare_batch") == 4
    img_ids, o, d, rgba = next(ds)
    assert bool((rgba[:, 3] == 1).all()) and int(img_ids.max()) < 50          # opaque JPEG frames


def test_reference_written_pkl_with_flushed_second_moments_keeps_training_finite(monkeypatch, tmp_path):
    """A params.pkl written by the REFERENCE holds fp16 Adam moments: second moments of the hash table (g^2 ~ 1e-10) flush to 0 while the
    first moment survives.  Loading such a file and training on must not blow entries up (lr * m / (sqrt(0) + 1e-15))."""
    from jnerf_b200.utils import ckpt_compat as cc
    r, _ = make_runner(monkeypatch, seed=5)
    for _ in range(4):
        r.train_step()
    p = str(tmp_path / "params.pkl")
    r.cfg.m_training_step = 5
    r.save_ckpt(p)
    ref = cc.read_reference_ckpt(p)
    pg = ref["nested_optimizer"]["defaults"]["param_groups"][0]
    for k in ("values_f32", "m_f32"):                              # what a reference-written file lacks
        del pg[k]
    del ref["ema_optimizer"]["defaults"]["param_groups"][0]["values_f32"]
    v16, m16 = np.asarray(pg["values"][0]), np.asarray(pg["m"][0])
    assert ((v16 == 0) & (m16 != 0)).any()                         # the hazard is really present in the fp16 copies
    cc.write_reference_ckpt(ref, p)
    r2, _ = make_runner(monkeypatch, seed=6)
    r2.load_ckpt(p)
    st = r2.optimizer._nested_optimizer.state[0]
    assert not ((st.v == 0) & (st.m != 0)).any()
    g_before = r2.model.pos_encoder.m_grid.detach().float().clone()
    for _ in range(3):
        assert torch.isfinite(r2.train_step()).all()
    g = r2.model.pos_encoder.m_grid.detach().float()
    assert torch.isfinite(g).all() and float((g - g_before).abs().max()) <= 3 * 0.1 + 1e-3      # |Adam update| <= lr per step


def test_runner_on_the_linear_fallback_model_renders_and_saves(monkeypatch, tmp_path):
    """The reference's own fallback (ngp_network.py:54-67: nn.Linear chains when the fused MLP is off): the Runner must still train
    through the per-operator path, render, compute PSNR and write / read a native checkpoint; the .pkl interchange format (fused
    parameter layout) and data-parallel training are refused with a clear error."""
    cpu_backend.install(monkeypatch)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**R.lego_cfg(fp16=True, synthetic=True, seed=2, n_rays_per_batch=64, target_batch_size=32768))
    cfg = get_cfg()
    cfg.model.fused = False
    cfg.model.use_fully = False
    cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W = 3, 16, 16
    cfg.dataset.val = None
    r = R.Runner()
    assert not r.fast and not hasattr(r.model.density_mlp, "con_weights")
    bits, _ = ol.sphere_bitfield(0.35, cascades=r.sampler.NERF_CASCADES)
    r.sampler.density_grid_bitfield.copy_(torch.from_numpy(bits[:r.sampler.density_grid_bitfield.numel()]))
    cfg.m_training_step = 1
    r.train(steps=2)
    img, tar = r.render_img("train", 0)
    assert img.shape == (16, 16, 3) and torch.isfinite(img).all() and np.isfinite(r.psnr("train", max_images=1))
    p = str(tmp_path / "ckpt.pt")
    r.save_ckpt(p)
    r.load_ckpt(p)
    with pytest.raises(NotImplementedError):
        r.save_ckpt(str(tmp_path / "params.pkl"))
    get_cfg().clear()
    update_cfg(**R.lego_cfg(fp16=True, synthetic=True, seed=2, n_rays_per_batch=64, target_batch_size=32768))
    cfg = get_cfg()
    cfg.model.fused = False
    cfg.model.use_fully = False
    cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W = 3, 16, 16
    cfg.dataset.val = None
    with pytest.raises(ValueError, match="data-parallel"):
        R.Runner(rank=0, world_size=2, process_group=None)


def test_host_fed_batches_equal_device_batches(monkeypatch):
    """Runner.train_step_host (pinned host batch -> staging slot on the copy stream -> train_step) gives the same step as train_step on
    the same batch, alternates its two staging slots, and does not copy a batch twice when it was announced as `next_batch`."""
    ra, fa = make_runner(monkeypatch, seed=8)
    rb, fb = make_runner(monkeypatch, seed=8)
    batches = [tuple(t.clone() for t in ra.next_batch()) for _ in range(3)]
    for b in batches:
        rb.next_batch()                                            # keep the two datasets' pixel streams aligned
    fb.calls.clear()                                               # (the second install replaced the operator layer for both runners)
    for k, b in enumerate(batches):
        la = ra.train_step(tuple(t.clone() for t in b))
        lh = rb.train_step_host(b, batches[k + 1] if k + 1 < len(batches) else None)
        assert abs(float(lh) - float(la.mean())) <= 1e-6 * max(1.0, abs(float(la.mean())))
    assert fb.calls.count("blend_target") == 6 and "prepare_batch" not in fb.calls
    assert torch.equal(ra.model.pos_encoder.m_grid.detach(), rb.model.pos_encoder.m_grid.detach())
    st = rb._host_stage
    assert st["k"] == 3 and st["slots"][0] is not None and st["slots"][1] is not None and st["staged"] == [None, None]


FRONT_OPS = ["prepare_batch", "march", "compact"]
BACK_OPS = ["network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema", "adam_ema", "adam_ema"]


def test_pipelined_steps_equal_sequential_steps(monkeypatch):
    """The software pipeline (front of step i+1 enqueued under step i) reorders launches, not arithmetic: same losses, parameters, ray
    batch adaptation and rng position as the sequential step, across a 16-step window edge (no prefetch into a step that opens with
    an occupancy-grid update; the ray batch adapts after the 16th march, before the next front)."""
    out = {}
    for pipe in (False, True):
        r, fake = make_runner(monkeypatch, seed=11, start_step=12, pipeline=pipe)
        assert (r._pipe is not None) == pipe
        # the grid update at step 16 evaluates 2 M densities in the scalar oracle: stand-in that only counts (its own test covers it)
        upd = []
        monkeypatch.setattr(r.sampler, "update_density_grid", lambda: upd.append(r.cfg.m_training_step))
        fake.calls.clear()
        losses, rays = [], []
        for k in range(7):                                          # steps 12 .. 18
            rays.append(r.sampler.n_rays_per_batch)
            n0 = len(fake.calls)
            losses.append(r.train_step().clone())
            if pipe:
                step = 12 + k
                first = k == 0 or step == 16                        # nothing was prefetched for these
                expect = (FRONT_OPS if first else []) + BACK_OPS + (FRONT_OPS if (step + 1) % 16 else [])
                assert fake.calls[n0:] == expect, (step, fake.calls[n0:])
        assert upd == [16]
        if pipe:
            assert r._pipe["pending"] is not None and r._pipe["pending"]["step"] == 19 and r._pipe["prefetched"] == 6
            r._pipe["pending"] = None
        out[pipe] = dict(losses=torch.stack([l.float().mean() for l in losses]), rays=rays, grid=r.model.pos_encoder.m_grid.detach().clone(),
                         w=r.model.rgb_mlp.con_weights.detach().clone(), n_step=r.optimizer._nested_optimizer.n_step, rng=r.sampler.rng.copy())
    a, b = out[False], out[True]
    assert a["rays"] == b["rays"] and a["rays"][4] != a["rays"][3]               # adapted after step 15's march, in both
    assert torch.equal(a["losses"], b["losses"]) and torch.equal(a["grid"], b["grid"]) and torch.equal(a["w"], b["w"])
    assert a["n_step"] == b["n_step"] == 7
    assert np.array_equal(ol.pcg32_advance(a["rng"].copy()), b["rng"])           # the pipelined run has marched step 19 already


def test_pipelined_checkpoint_and_evaluation_between_steps(monkeypatch, tmp_path):
    """With a prefetched front pending: a checkpoint stores the jitter-stream position of its global_step (not the prefetched one),
    loading a checkpoint drops the front, and the evaluation renderer leaves it intact for the next step."""
    r, fake = make_runner(monkeypatch, seed=13, pipeline=True)
    rng0 = r.sampler.rng.copy()
    for _ in range(3):
        r.train_step()
    assert r._pipe["pending"]["step"] == 4
    assert np.array_equal(r.sampler.rng, ol.pcg32_advance(rng0.copy(), 4 << 32))   # four marches done
    p = str(tmp_path / "ckpt.pt")
    r.save_ckpt(p)
    ck = torch.load(p, weights_only=True)
    assert np.array_equal(ck["sampler"]["rng"].numpy().astype(np.uint64), ol.pcg32_advance(rng0.copy(), 3 << 32)) and ck["global_step"] == 4
    pend = r._pipe["pending"]
    img, _ = r.render_img_nosync("train", 0)
    assert r._pipe["pending"] is pend and torch.isfinite(img).all()
    fake.calls.clear()
    r.train_step()
    assert fake.calls[:len(BACK_OPS)] == BACK_OPS                                  # consumed the prefetched front
    r.load_ckpt(p)
    assert r._pipe["pending"] is None and r.cfg.m_training_step == 4
    fake.calls.clear()
    r.train_step()
    assert fake.calls[:len(FRONT_OPS)] == FRONT_OPS


def test_pipelined_host_fed_batches(monkeypatch):
    """train_step_host with next_batch: the next batch's blend + march are enqueued under the current step; same result as feeding the
    batches one by one without announcing the next."""
    out = {}
    for announce in (False, True):
        r, fake = make_runner(monkeypatch, seed=17, pipeline=True)
        ds = r.dataset["train"]
        batches = []
        for k in range(4):
            pix = ds.next_pixels(64)
            img_ids, o, d = ds.rays_for(pix)
            batches.append((img_ids.clone(), o.clone(), d.clone(), ds.rgba_for(pix).clone()))
        fake.calls.clear()
        ls = []
        for k in range(4):
            n0 = len(fake.calls)
            ls.append(float(r.train_step_host(batches[k], batches[k + 1] if announce and k < 3 else None).item()))
            if announce:
                front = ["blend_target", "march", "compact"]
                assert fake.calls[n0:] == (front if k == 0 else []) + BACK_OPS + (front if k < 3 else []), fake.calls[n0:]
        out[announce] = (ls, r.model.pos_encoder.m_grid.detach().clone())
    assert out[False][0] == out[True][0] and torch.equal(out[False][1], out[True][1])


def test_pipelined_front_is_dropped_when_the_caller_changes_course(monkeypatch):
    """A prefetched front that no longer matches the next call (another batch is fed, or the step counter was moved) is discarded and a
    fresh one is made on the spot; training goes on."""
    r, fake = make_runner(monkeypatch, seed=19, pipeline=True)
    ds = r.dataset["train"]
    r.train_step()
    assert r._pipe["pending"] is not None and r._pipe["pending"]["src"] is None
    pix = ds.next_pixels(64)
    img_ids, o, d = ds.rays_for(pix)
    fake.calls.clear()
    loss = r.train_step((img_ids, o, d, ds.rgba_for(pix)))           # a fed batch instead of the device-generated one that was prefetched
    assert fake.calls[:3] == ["blend_target", "march", "compact"] and torch.isfinite(loss).all()
    assert r._pipe["pending"] is None                                # the caller did not say which batch comes next
    r.train_step()
    r.cfg.m_training_step += 5                                       # e.g. a resumed schedule
    fake.calls.clear()
    assert torch.isfinite(r.train_step()).all() and fake.calls[:3] == FRONT_OPS


def test_two_rank_ray_batch_adapts_globally_across_a_window_edge(tmp_path):
    """Steps 12 .. 17 on two gloo ranks, sequential and pipelined: at the end of step 15 the GLOBAL ray batch (2 x 32 rays) is adapted to
    the global 16-step sample count against the global budget with the reference's formula (rounded to 128 rays), and every rank takes
    half of it -- identically on both ranks and in both step orders (the pipelined runner all-reduces and reads the counter back on
    its side stream); the replicas stay identical across the edge."""
    import os
    import torch.multiprocessing as mp
    out = {}
    for pipe in (False, True):
        ret = mp.Manager().dict()
        mp.spawn(_dp_worker, args=(2, 29715 + int(pipe) + os.getpid() % 1000, str(tmp_path), ret, pipe, 12, 6), nprocs=2, join=True)
        a, b = ret[0], ret[1]
        assert a["rays"] == b["rays"] and a["rays"][:4] == [32] * 4 and a["rays"][4] != 32          # adapted after step 15's march
        assert (2 * a["rays"][4]) % 128 == 0                                                          # the GLOBAL batch is rounded, not the shard
        assert a["table_sum"] == b["table_sum"] and np.array_equal(a["w"], b["w"])
        out[pipe] = (a["rays"], a["losses"], a["table_sum"])
    assert out[False] == out[True]
