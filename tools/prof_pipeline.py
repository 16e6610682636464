"""Per-kernel device time of pipelined training steps of the bench workload (lego, synthetic, 2^18 samples a step), from
torch.profiler CUDA activity: `steps` steps after `pre` untimed steps, then the same stages run alone on one stream (bench.py's
stage split) for the standalone times.  Prints one JSON line:

  pipelined / alone  -- per kernel name: launches and us per step
  overlap            -- per step, how long a march kernel of the next step's front ran while network_bwd256_kernel ran
  fwd_wait_us        -- per step, how long the main stream sat idle before the network forward because the front had not finished

  python tools/prof_pipeline.py [--pre 256] [--steps 100] [--out DIR]     (the trace goes to DIR/pipeline.pt.trace.json)"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def kernels(trace_path):
    ev = json.load(open(trace_path))["traceEvents"]
    return sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])


def per_step(ks, steps):
    out = {}
    for k in ks:
        name = k["name"].replace("(anonymous namespace)::", "").replace("void ", "")
        d = out.setdefault(name.split("(")[0].split("<")[0], [0, 0.0])
        d[0] += 1
        d[1] += k["dur"]
    return {n: {"launches": c, "us_per_step": t / steps} for n, (c, t) in sorted(out.items(), key=lambda kv: -kv[1][1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pre", type=int, default=256)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default="profiles")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    import bench

    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=1, target_batch_size=1 << 18))
    cfg = get_cfg()
    cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W, cfg.dataset.val = 100, 800, 800, None
    cfg.dataset.train.pop("root_dir", None)
    r = Runner()
    for _ in range(args.pre):
        r.train_step()
    torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "pipeline.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(args.steps):
            r.train_step()
        torch.cuda.synchronize()
    p.export_chrome_trace(path)
    ks = kernels(path)
    with profile(activities=[ProfilerActivity.CUDA]) as p2:
        bench.stage_times(r, 16)
        torch.cuda.synchronize()
    path2 = os.path.join(args.out, "alone.pt.trace.json")
    p2.export_chrome_trace(path2)

    bwd = [k for k in ks if "network_bwd256_kernel" in k["name"]]
    fwd = [k for k in ks if "network_fwd_kernel" in k["name"]]
    march = [k for k in ks if "march_" in k["name"]]
    overlap = []
    for b in bwd:
        b0, b1 = b["ts"], b["ts"] + b["dur"]
        overlap.append(sum(max(0.0, min(b1, m["ts"] + m["dur"]) - max(b0, m["ts"])) for m in march))
    # main-stream idle time in front of each forward: the gap to the latest kernel that ended before it on the forward's stream
    waits = []
    for f in fwd:
        prev = [k["ts"] + k["dur"] for k in ks if k["args"].get("stream") == f["args"].get("stream") and k["ts"] < f["ts"]]
        if prev:
            waits.append(max(0.0, f["ts"] - max(prev)))
    res = {"pipe_at": r._pipe["at"] if r._pipe else None, "steps": args.steps,
           "rays_per_batch": r.sampler.n_rays_per_batch,
           "pipelined": per_step(ks, args.steps), "alone": per_step(kernels(path2), 16),
           "bwd_us": sorted(b["dur"] for b in bwd)[len(bwd) // 2] if bwd else None,
           "march_under_bwd_us_median": sorted(overlap)[len(overlap) // 2] if overlap else None,
           "fwd_wait_us_median": sorted(waits)[len(waits) // 2] if waits else None,
           "fwd_wait_us_mean": sum(waits) / len(waits) if waits else None}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
