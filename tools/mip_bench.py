#!/usr/bin/env python
"""Mip-NeRF training step on the H100: the fused MipNerfMLP kernels (ops.mip_fwd + one ops.nerf_bwd over both levels) against the same
network as fp16 torch.nn.Linear + autograd (cuBLAS), both around the same sampler kernels (mip_sample, mip_resample, mip_composite_fwd,
mip_composite_loss_bwd) and Adam.  Per step: the time of every stage from CUDA events, and the whole step.  Rays per step: 288 (mip_base.py's
batch) and 4096; 128 samples a level.  --degs 16 times the network at multicam.py's 16 IPE degrees (96 encoding columns; multicam.py's
batch is --rays 3072).  Prints one JSON line with the GPU's name, power limit and SM clock.

    python tools/mip_bench.py [--steps 50] [--warmup 5] [--rays 288 4096] [--degs 8]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jnerf_b200 import ops, plugin  # noqa: E402,F401
from jnerf_b200.mip_runner import mip_cfg  # noqa: E402
from jnerf_b200.plugin import mip  # noqa: E402
from jnerf_b200.utils.config import get_cfg, update_cfg  # noqa: E402

STAGES = ("sample", "fwd_coarse", "composite", "resample", "fwd_fine", "loss_bwd", "net_bwd", "adam")


def make(fused, degs, seed=1):
    get_cfg().clear()
    update_cfg(**mip_cfg(using_fp16=fused, seed=seed, max_deg_point=degs))
    m = mip.MipNerfMLP()
    return m if fused else m.half()


def step(m, fused, rays, target, rng, saved, ev, degs):
    S, R = 128, rays.shape[0]
    n = R * S
    cfg = get_cfg()
    p, bias = cfg.rgb_padding, cfg.density_bias
    ev[0].record()
    t_c = ops.mip_sample(rays, S, False, True, rng)
    ev[1].record()
    if fused:
        raw = torch.empty((2 * n, 4), dtype=torch.float16, device="cuda")
        half = saved.numel() // 2
        ops.mip_fwd(rays, t_c, m.params, out=raw[:n], saved=saved[:half], degs=degs)
        raw_c = raw[:n]
    else:
        enc, view = ops.mip_encode(rays, t_c, degs=degs)
        raw_c = m.execute(enc.half(), view.half())
    ev[2].record()
    w = ops.mip_composite_fwd(raw_c.detach(), t_c, rays, p, bias, False)[3]
    ev[3].record()
    t_f = ops.mip_resample(t_c, w, 0.01, True, rng)
    ev[4].record()
    if fused:
        ops.mip_fwd(rays, t_f, m.params, out=raw[n:], saved=saved[half:], degs=degs)
    else:
        enc, view = ops.mip_encode(rays, t_f, degs=degs)
        raw_f = m.execute(enc.half(), view.half())
        raw = torch.cat([raw_c.detach(), raw_f.detach()])
    ev[5].record()
    _, _, draw = ops.mip_composite_loss_bwd(raw, torch.cat([t_c, t_f]), rays, target, None, p, bias, False, 0.1, grad_scale=float(R))
    ev[6].record()
    if fused:
        grads = [ops.mip_bwd(m.params, saved, draw, degs)]
    else:
        torch.autograd.backward([raw_c, raw_f], [draw[:n], draw[n:]])
        grads = [q.grad for q in m.parameters()]
    ev[7].record()
    for q, g, st in zip(m.parameters(), grads, m._adam):
        ops.adam_ema(q.data.view(-1), g.reshape(-1), *st, 1e-3, 1, 0.9, 0.99, 1e-15, 0.0, grad_scale=1.0 / R, zero_grad=False)
        q.grad = None
    ev[8].record()


def run(fused, R, steps, warmup, degs=8):
    m = make(fused, degs)
    m._adam = [tuple(torch.zeros(q.numel(), dtype=torch.float32, device="cuda") for _ in range(2)) + (q.detach().float().reshape(-1).clone(),)
               for q in m.parameters()]
    g = torch.Generator(device="cuda").manual_seed(0)
    o = (torch.rand((R, 3), device="cuda", generator=g) - 0.5) * 8
    d = torch.nn.functional.normalize(-o + torch.randn((R, 3), device="cuda", generator=g) * 0.3, dim=-1)
    rays = torch.cat([o, d, d, torch.full((R, 1), 1.2e-3, device="cuda"), torch.full((R, 1), 2.0, device="cuda"),
                      torch.full((R, 1), 6.0, device="cuda")], -1).contiguous()
    target = torch.rand((R, 3), device="cuda", generator=g)
    saved = torch.empty(2 * ops.mip_workspace_bytes(R * 128, degs)[0], dtype=torch.uint8, device="cuda") if fused else None
    rng = ops.pcg32_seed(1)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
    acc = dict.fromkeys(STAGES, 0.0)
    for i in range(warmup + steps):
        step(m, fused, rays, target, rng, saved, ev, degs)
        ops.pcg32_advance(rng, 2 * R * 129)
        torch.cuda.synchronize()
        if i >= warmup:
            for k, name in enumerate(STAGES):
                acc[name] += ev[k].elapsed_time(ev[k + 1]) / steps
    acc["step"] = sum(acc[k] for k in STAGES)
    return {k: round(v, 4) for k, v in acc.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rays", type=int, nargs="+", default=[288, 4096])
    ap.add_argument("--degs", type=int, default=8, choices=(8, 16))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mip_bench.py measures on the GPU: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(), "samples_per_level": 128, "ipe_degs": a.degs, "ms": {}}
    for R in a.rays:
        fused, chain = run(True, R, a.steps, a.warmup, a.degs), run(False, R, a.steps, a.warmup, a.degs)
        res["ms"][str(R)] = {"fused": fused, "cublas_fp16": chain, "step_speedup": round(chain["step"] / fused["step"], 3),
                             "network_speedup": round((chain["fwd_coarse"] + chain["fwd_fine"] + chain["net_bwd"])
                                                      / (fused["fwd_coarse"] + fused["fwd_fine"] + fused["net_bwd"]), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
