#!/usr/bin/env python
"""bench.py -- Instant-NGP lego training throughput on N H100s (BASELINE.json metric: NGP lego iters/s & rays/s).

  python bench.py --gpus N --steps K --warmup W            our arm   (torchrun for N>1: one rank per GPU, NCCL)
  python bench.py --impl reference --gpus N --steps K ...  reference arm: the path's CPU implementation (oracle port)
  python bench.py ... --dump-outputs DIR                   also write what the last timed step computed to DIR/<name>.npy

A step = one full training iteration of projects/ngp/configs/ngp_base.py + fp16 (BASELINE config #2):
[density-grid update every 16] -> ray gen -> march -> fused hash+MLP forward -> composite + Huber + composite
backward -> fused MLP/hash backward -> [grad all-reduce] -> fused Adam+EMA over all 12.2 M parameters.
On the device the steps are software-pipelined (jnerf_b200/runner.py: ray gen + march of step i+1 run on a second stream under step
i's network kernels and optimizer sweep; NGP_PIPELINE=0 gives the strictly sequential step): the timed region holds K complete
steps either way, nothing is skipped or cached.
Data is synthetic (lego is downloaded at run time by the reference and is not available offline): 100 procedurally
ray-traced 800x800 RGBA views with lego's intrinsics; weights are random-init.  Before the W warm-up steps the model is
trained for --pretrain steps (untimed) so that the occupancy grid and the adaptive ray batch are in steady state, which
is also the state the reference's published tqdm reading (133 it/s) refers to.

value  = rays/s over all ranks, inputs resident in HBM (pixels shuffled and rays generated on the device, as the
         reference does);  e2e = the same metric with every step's ray batch (origins, directions, RGBA targets)
         copied from pinned host memory and the loss read back, through Runner.train_step_host(batch, next_batch): the
         copies run on the Runner's copy stream inside the timed region, the next batch's under the current step.
Prints ONE JSON line on rank 0."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ALGO = {   # algorithmic bytes / flops per sample (SURVEY.md 8d, DESIGN.md)
    "network_fwd": dict(bytes=524 + 28 + 8 + 64, flops=20480),
    "network_bwd": dict(bytes=64 + 28 + 8 + 128 * 8, flops=61440),
}


def peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return p["hbm_gbs"], p["bf16_tflops"], "measured"
    except Exception:
        return 3350.0, 989.0, "H100 SXM data sheet (HBM3, dense BF16)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 20 ms from before the warm-up; samples inside the timed region are kept."""
    Q = "timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index=0):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "20", "-i", str(self.index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=lambda: [self.lines.append(l) for l in self.proc.stdout], daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def mark(self):
        """Host time stamp (same clock nvidia-smi prints) -- used to pick the samples that fall inside the timed region."""
        return time.time()

    def stop(self, t0=None, t1=None):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.05)
        self.proc.terminate()
        self.t.join(timeout=2)
        import datetime
        rows = []
        for l in self.lines:
            f = [x.strip() for x in l.split(",")]
            if len(f) < 9:
                continue
            try:
                ts = datetime.datetime.strptime(f[0], "%Y/%m/%d %H:%M:%S.%f").timestamp()
                rows.append((ts, float(f[1]), float(f[2]), f[5:9]))
            except ValueError:
                continue
        inside = [r for r in rows if t0 is not None and t0 <= r[0] <= t1]
        window = "timed region"
        if len(inside) < 3:                       # nvidia-smi samples slower than asked on some boxes: fall back to everything under load
            inside, window = rows, "warm-up + timed region"
        sm, mx, reasons = [], [], set()
        for _, a, b, flags in inside:
            sm.append(a); mx.append(b)
            f = [None] * 5 + list(flags)
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons), "samples": len(sm),
                "window": window}


# ---------------------------------------------------------------------------------------------------- CPU arm
def cpu_train_iteration(n_rays, seed=0):
    """One training iteration's ray-proportional work with the oracle (CPU port of the reference path): march, compaction,
    hash encode + MLPs forward, composite + Huber + composite backward, MLP backward, hash scatter.  Returns seconds, rays, samples."""
    import numpy as np
    import oracle_lib as ol
    cfg = ol.HashCfg(1)
    rng = np.random.default_rng(seed)
    st = cpu_train_iteration.__dict__
    if "grid" not in st:
        st["grid"] = rng.uniform(-1e-4, 1e-4, cfg.n_params).astype(np.float16)
        st["wd"] = rng.uniform(-0.3, 0.3, 3072).astype(np.float16)
        st["wr"] = rng.uniform(-0.3, 0.3, 7168).astype(np.float16)
        st["bits"], _ = ol.sphere_bitfield(0.3, shell=0.02)      # thin shell: ~60-90 samples per hit ray, like a trained scene
    grid, wd, wr, bits = st["grid"], st["wd"], st["wr"], st["bits"]
    o, d = ol.random_rays(n_rays, seed=seed)
    bg = rng.random((n_rays, 3), dtype=np.float32)
    target = rng.random((n_rays, 3), dtype=np.float32)
    t0 = time.perf_counter()
    coords, _, numsteps, cnt = ol.march(o, d, bits, max_samples=n_rays * 1024)
    S = int(cnt[1])
    cc, ns_c, _ = ol.compact(coords, numsteps, max(S, 1))
    pos, dirs = np.ascontiguousarray(cc[:S, :3]), np.ascontiguousarray(cc[:S, 4:])
    out, enc, h = ol.network_fwd(cfg, pos, dirs, grid, wd, wr, acc32=False)
    rgb = ol.composite_fwd(out, cc, numsteps, ns_c, bg)
    g, _ = ol.huber_grad(rgb, target)
    dnet = ol.composite_bwd(out, cc, ns_c, g.reshape(n_rays, 3), rgb, 0.001)
    _, inter_d = ol.mlp_fwd(wd, enc, 0)
    rin = np.concatenate([h, ol.sh(dirs, np.float16)], 1)
    _, inter_r = ol.mlp_fwd(wr, rin, 1)
    dYr = np.zeros((S, 16), np.float16)
    dYr[:, :3] = dnet[:, :3]
    d_rin, _, _ = ol.mlp_bwd(wr, rin, inter_r, dYr, 1, 3)
    dYd = d_rin[:, :16].astype(np.float32)
    dYd[:, 0] += dnet[:, 3].astype(np.float32)
    d_enc, _, dWd = ol.mlp_bwd(wd, enc, inter_d, dYd.astype(np.float16), 0, 16)
    gg = ol.hash_bwd(cfg, pos, d_enc)
    # dense Adam + EMA over all 12.2 M parameters, as the reference's optimizer does every step (optims/adam.py, optims/ema.py)
    if "opt" not in st:
        st["opt"] = [dict(p=p, m=np.zeros(p.size, np.float32), v=np.zeros(p.size, np.float32), master=p.astype(np.float32)) for p in (grid, wd, wr)]
        st["step"] = 0
    st["step"] += 1
    for o, g in zip(st["opt"], (gg, dWd, np.zeros(wr.size, np.float32))):
        ol.adam_ema(o["p"], np.ascontiguousarray(g, np.float32), o["m"], o["v"], o["master"], 1e-2, st["step"])
    return time.perf_counter() - t0, n_rays, S


def cpu_baseline(n_rays=256, iters=6):
    for _ in range(2):
        cpu_train_iteration(64)                             # warm up (builds the oracle, touches the table and the optimizer state)
    rates, s = [], 0
    for k in range(iters):
        dt, rr, ss = cpu_train_iteration(n_rays, seed=k + 1)
        rates.append(rr / dt)
        s += ss
    rates.sort()
    cores = len(os.sched_getaffinity(0))
    return {"value": rates[len(rates) // 2], "unit": "rays/s", "cores": cores, "kind": "port",
            "sample": f"median of {iters} full training iterations of {n_rays} rays ({s // iters} samples each): march, hash+MLP fwd, "
                      f"composite+loss+bwd, MLP bwd, hash scatter, dense Adam+EMA over all 12.2 M parameters, with the oracle "
                      f"(OpenMP where the loop is parallel)",
            "spread": [rates[0], rates[-1]]}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    # torchrun exports OMP_NUM_THREADS=1 to every rank; this arm is the CPU implementation with all the host threads it can
    # use, and libgomp reads the variable when the oracle library is loaded (inside cpu_train_iteration)
    os.environ["OMP_NUM_THREADS"] = str(len(os.sched_getaffinity(0)))
    n_rays = max(64, min(256, 16384 // max(args.steps, 1)))    # bounded sample: the whole run stays within minutes
    for _ in range(max(args.warmup, 2)):
        cpu_train_iteration(64)
    t, r, s, rates = 0.0, 0, 0, []
    for k in range(args.steps):
        dt, rr, ss = cpu_train_iteration(n_rays, seed=k + 1)
        t, r, s = t + dt, r + rr, s + ss
        rates.append(rr / dt)
    cores = len(os.sched_getaffinity(0))
    rates.sort()
    v = rates[len(rates) // 2]                                # median over the steps: robust against a noisy neighbour on the shared host
    print(json.dumps({
        "impl": "reference", "metric": "ngp_lego_train_rays_per_s", "value": v, "unit": "rays/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": t / args.steps * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f16", "data": "synthetic", "config": {"workload": "Instant-NGP lego (ngp_base.py + fp16), synthetic stand-in scene; "
                                                        f"bounded sample of {n_rays} rays per step on the host CPU"},
        "cpu_baseline": {"value": v, "unit": "rays/s", "cores": cores, "kind": "port",
                         "sample": f"median of {args.steps} full iterations x {n_rays} rays (~{s // max(args.steps, 1)} samples each, dense Adam+EMA "
                                   f"included), oracle port of the reference path", "spread": [rates[0], rates[-1]]},
        "e2e": {"value": v, "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}))


# ---------------------------------------------------------------------------------------------------- our arm
def run_ours(args):
    import torch
    import torch.distributed as dist
    from jnerf_b200 import lib, ops, plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    pg = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        pg = dist.group.WORLD
    lib.load()
    get_cfg().clear()
    fox = args.workload == "fox"
    update_cfg(**(fox_cfg if fox else lego_cfg)(fp16=True, synthetic=True, seed=1, target_batch_size=args.target_batch))
    cfg = get_cfg()
    if fox:                                # BASELINE config #3: the capture's own frame count / resolution unless overridden
        if args.images != 100:
            cfg.dataset.train.n_images = args.images
        if args.res != 800:
            cfg.dataset.train.W, cfg.dataset.train.H = args.res, args.res * 16 // 9
    else:
        cfg.dataset.train.n_images = args.images
        cfg.dataset.train.H = cfg.dataset.train.W = args.res
    cfg.dataset.val = None
    cfg.dataset.train.pop("root_dir", None)
    if args.data_dir:                      # a real capture in the reference's layout (transforms*.json + images), e.g. data/lego or data/fox
        cfg.dataset.train = dict(type="NerfDataset", root_dir=args.data_dir, batch_size=4096, mode="train")
    runner = Runner(rank=rank, world_size=world, process_group=pg)
    ds0 = runner.dataset["train"]
    n_img, res_txt = ds0.n_images, f"{ds0.W}x{ds0.H}"

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()                    # started early: nvidia-smi needs a few hundred ms before its first sample
    # steady state: occupancy grid carved, ray batch adapted (untimed)
    for _ in range(args.pretrain):
        runner.train_step()
    for _ in range(args.warmup):
        runner.train_step()
    sync()

    # ---- timed region: K steps, device-resident inputs ----
    launches0 = lib.launch_count
    rays = 0
    sync()
    profiling = bool(os.environ.get("NGP_PROFILE"))          # ncu --profile-from-start off: capture exactly the timed region
    if profiling:
        torch.cuda.profiler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_host0 = clocks.mark()
    e0.record()
    loss = None
    for _ in range(args.steps):
        rays += runner.sampler.n_rays_per_batch
        loss = runner.train_step()
    runner._table_ready()                 # N>1: the last step's all-gather belongs to the timed region
    e1.record()
    sync()
    t_host1 = clocks.mark()
    if profiling:
        torch.cuda.profiler.stop()
    if args.dump_outputs and rank == 0:               # after the clock window: the copies to the host are not part of the timed steps
        dump_outputs(runner, loss, args.dump_outputs)
    ms = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    launches = lib.launch_count - launches0
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    clk = clocks.stop(t_host0, t_host1) if rank == 0 else None
    total_rays = rays * world
    value = total_rays / (ms * 1e-3)

    # ---- e2e: every step's ray batch comes from pinned host memory; loss goes back to the host ----
    ds = runner.dataset["train"]
    host_batches = []
    for _ in range(min(args.steps, 64) + 1):
        b = runner.next_batch()
        host_batches.append(tuple(t.cpu().pin_memory() for t in b))
    h2d = sum(t.numel() * t.element_size() for t in host_batches[0])

    R_e2e, ds_e2e = runner.sampler.n_rays_per_batch, runner.dataset["train"]

    def host_step(k):
        # the user-facing call for host-fed batches: this step's batch and (for overlap) the next one, both in pinned host memory;
        # the H2D copies and the D2H of the mean loss run on the Runner's copy stream inside the timed region
        hb = host_batches[k % len(host_batches)]
        loss_host = runner.train_step_host(hb, host_batches[(k + 1) % len(host_batches)])
        # the pre-generated batches keep their size: do not let the 16-step adaptation run away from them
        runner.sampler.n_rays_per_batch = ds_e2e.batch_size = R_e2e
        return hb[1].shape[0]

    for k in range(max(args.warmup, 3)):
        host_step(k)
    sync()
    rays_e = 0
    e0.record()
    for k in range(args.steps):
        rays_e += host_step(k)
    runner._table_ready()
    e1.record()
    sync()
    ms_e = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    if world > 1:
        dist.all_reduce(ms_e, op=dist.ReduceOp.MAX)
    ms_e = float(ms_e.item())
    e2e = {"value": rays_e * world / (ms_e * 1e-3), "unit": "rays/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
           "iters_per_s": args.steps / (ms_e * 1e-3)}

    # ---- per-kernel times on the launching stream (CUDA events), for the roofline of the dominant kernel ----
    stage = stage_times(runner, 16)
    n_samples = stage.pop("_samples")
    hbm, tfl, src = peaks()
    dom = max(("network_fwd", "network_bwd"), key=lambda k: stage[k])
    algo = dict(ALGO[dom])
    t_dom = stage[dom] * 1e-3
    gbs = n_samples * algo["bytes"] / t_dom / 1e9
    roofline = {"kernel": dom, "bound": "hbm", "achieved": gbs, "peak": hbm, "unit": "GB/s", "frac": gbs / hbm,
                "peak_source": src, "launch_ms": stage[dom], "samples_per_launch": n_samples,
                "algorithmic_bytes_per_sample": algo["bytes"],
                "tensor": {"achieved_tflops": n_samples * algo["flops"] / t_dom / 1e12, "peak_tflops": tfl,
                           "frac": n_samples * algo["flops"] / t_dom / 1e12 / tfl},
                "stage_ms": stage}
    out = {
        "metric": f"ngp_{args.workload}_train_rays_per_s", "value": value, "unit": "rays/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None, "dtype": "f16",
        "data": f"real: {args.data_dir}" if args.data_dir else "synthetic",
        "iters_per_s": args.steps / (ms * 1e-3), "published_iters_per_s_rtx3090": 133.0, "samples_per_s": None,
        "config": {"workload": ("Instant-NGP fox: projects/ngp/configs/ngp_fox.py (BASELINE config #3: aabb_scale 4, cone stepping, fp16 fully-fused MLP), "
                                if fox else "Instant-NGP lego: projects/ngp/configs/ngp_base.py + fp16 fully-fused MLP (BASELINE config #2), ") +
                               f"{n_img} {'real' if args.data_dir else 'synthetic'} {res_txt} views, target_batch_size {args.target_batch} samples/iter/GPU"
                               f"{' (2^18)' if args.target_batch == 1 << 18 else ''}, adaptive ray batch "
                               f"({runner.sampler.n_rays_per_batch} rays/iter/GPU at measurement), pretrain {args.pretrain} steps",
                   "parallelism": f"dp{world}", "target_batch_size": args.target_batch,
                   "l2": "per-step working set (24 MB table + 171 MB optimizer state + 7 MB samples) exceeds the 50 MB L2; no explicit flush",
                   "step_pipeline": ({"enabled": True, "front_starts_at": runner._pipe["at"], "fronts_prefetched": int(runner._pipe["prefetched"]),
                                      "note": "ray generation + march of step i+1 on a second stream under step i's network kernels / optimizer sweep; "
                                              "every timed step contains one front and one back"}
                                     if getattr(runner, "_pipe", None) is not None else {"enabled": False}),
                   "cuda_graphs": {"enabled": bool(getattr(runner, "_graphs_enabled", False)), "graphs": len(getattr(runner, "_graphs", {}) or {}),
                                   "replays": int(getattr(runner, "graph_replays", 0))}},
        "e2e": e2e, "gpu_launches": launches, "clocks": clk, "roofline": roofline,
    }
    if rank == 0:
        out["samples_per_s"] = n_samples * world * out["iters_per_s"]
        if world == 1 and not args.no_cpu_baseline:
            out["cpu_baseline"] = cpu_baseline()
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def dump_outputs(runner, loss, out_dir):
    """Writes what the timed path hands its caller after the last timed step: that step's loss (Runner.train_step's return value)
    and the trained parameters, as float32 DIR/<name>.npy.  A parameter of more than 2^20 entries (the hash grid) is sampled at a
    fixed, seeded set of indices, so the files stay small and two builds can be compared entry for entry."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"loss": loss}
    arrays.update({f"param.{k}": v for k, v in runner.model.state_dict().items()})
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy().ravel()
        if a.size > 1 << 20:
            a = a[np.sort(np.random.default_rng(0).choice(a.size, 1 << 20, replace=False))]
        np.save(os.path.join(out_dir, name + ".npy"), a)


def stage_times(runner, iters):
    """Average per-stage device time (ms) of the training step, CUDA events on the current stream.  All `iters` iterations are
    enqueued before the one synchronisation: the GPU then always has a backlog, so an interval between two events is the device
    time of that stage and not the host's launch latency (a per-iteration sync inflated the stages made of many small launches)."""
    import torch
    from jnerf_b200 import ops
    s = runner.sampler
    names = ["prepare_batch", "march", "network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema"]
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)] for _ in range(iters)]
    n_dev = None
    if hasattr(runner, "_sync_front"):
        runner._sync_front()                             # a prefetched front of the step pipeline shares the march workspace with s.sample()
    for ev in evs:
        while runner.cfg.m_training_step % 16 in (0, 15):    # keep grid updates and the ray-batch adaptation (.item() sync) out of the split
            runner.cfg.m_training_step += 1
        ev[0].record()
        ds = runner.dataset["train"]
        R = s.n_rays_per_batch
        runner._table_ready()
        pix = ds.next_pixels(R)
        bg = torch.rand((R, 3), device="cuda")
        img_ids, rays_o, rays_d, target = ops.prepare_batch(pix.contiguous(), ds.W, ds.H, ds.transforms_gpu, ds.focal_lengths, ds.principal,
                                                            ds.image_data, bg)
        ev[1].record()
        s.sample(img_ids, rays_o, rays_d, is_training=True)
        ev[2].record()
        coords, n_dev = s.coords_compacted, s.n_samples_dev
        runner.net_forward(coords, n_dev)
        ev[3].record()
        ops.composite_loss_bwd(runner.net_out, coords, s._rays_numsteps, s._rays_numsteps_compacted, bg, target, s.density_grid_mean,
                               delta=0.1, cascades=s.NERF_CASCADES, dnet=runner.dnet)
        ev[4].record()
        runner.net_backward(coords, n_dev)
        ev[5].record()
        adam = runner.optimizer._nested_optimizer
        runner._optimizer_step(0.0, max(adam.n_step, 1))     # lr 0: timing only, parameters barely move; N>1: + reduce-scatter / all-gather
        runner._table_ready()
        ev[6].record()
        runner.cfg.m_training_step += 1
    torch.cuda.synchronize()
    out = {name: sum(ev[k].elapsed_time(ev[k + 1]) for ev in evs) / iters for k, name in enumerate(names)}
    out["_samples"] = min(int(n_dev.item()), s.target_batch_size)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=None, help="timed steps (default 1000; 32 for --impl reference)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--pretrain", type=int, default=256)
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--res", type=int, default=800)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--workload", default="lego", choices=["lego", "fox"],
                    help="lego = BASELINE config #2 (the headline line); fox = config #3 (aabb_scale 4, cone stepping) on its synthetic stand-in")
    ap.add_argument("--data-dir", default=None, help="train on a real capture in the reference's dataset layout instead of the synthetic stand-in")
    ap.add_argument("--target-batch", type=int, default=1 << 18,
                    help="target_batch_size, samples per iteration per GPU (ngp_base.py:75); BASELINE config #5 sweeps 2^16 .. 2^22 (tools/sweep.py)")
    ap.add_argument("--scaling", default="weak", choices=["weak", "strong"],
                    help="weak: --target-batch samples per iteration PER GPU (the default); strong: --target-batch is the GLOBAL "
                         "sample budget of an iteration, split evenly over the GPUs")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write the last step's loss and the trained parameters (the hash grid sampled) to DIR/<name>.npy; "
                         "inputs are seeded and the training step is deterministic, so the same arguments give the same files")
    args = ap.parse_args()
    if args.scaling == "strong":
        args.target_batch_global = args.target_batch
        args.target_batch = max(1 << 12, args.target_batch // max(1, int(os.environ.get("WORLD_SIZE", "1"))))
    if args.steps is None:
        args.steps = 32 if args.impl == "reference" else 1000
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
