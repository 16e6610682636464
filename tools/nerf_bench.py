"""Vanilla NeRF (nerf_cfg / projects/nerf/configs/nerf_base.py) on the GPU: one JSON line with
  * the card and its power limit,
  * ms per training step of nerf_cfg on the synthetic lego stand-in (ray batch adapted towards 2^18 samples a step),
  * forward and backward times at 2^18 rows of the fused kernels (csrc/nerf_mlp.cu) and of the same network as an fp16
    torch.nn.Linear + autograd chain (cuBLAS), on the same weights and rows, alternated, median and spread,
  * achieved TFLOP/s from the FLOP count below.

    python tools/nerf_bench.py [--rows 262144] [--reps 20] [--steps 200] [--out results/nerf_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (in, out) of every matrix product of one sample, as in ori_nerf_network.py: trunk, alpha, feature, views, rgb
LAYERS = [(63, 256)] + [(256, 256)] * 4 + [(319, 256)] + [(256, 256)] * 2 + [(256, 1), (256, 256), (283, 128), (128, 3)]
FWD_FLOP = sum(2 * i * o for i, o in LAYERS)                      # 1.19 M
# backward: weight gradients of every layer, data gradients of every layer but the first (no gradient into the encoding)
BWD_FLOP = sum(2 * i * o for i, o in LAYERS) + sum(2 * i * o for i, o in LAYERS[1:])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]))
    return out


def stats(ms):
    a = np.asarray(ms)
    return dict(median_ms=round(float(np.median(a)), 4), min_ms=round(float(a.min()), 4), max_ms=round(float(a.max()), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 18)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/nerf_bench.py measures on the GPU"
    from jnerf_b200 import ops, plugin  # noqa: F401
    from jnerf_b200.plugin import nerf
    from jnerf_b200.runner import Runner, nerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg

    get_cfg().clear()
    update_cfg(**nerf_cfg(fp16=True, synthetic=True, seed=1))
    N = args.rows
    P = nerf.pack(nerf.init_reference_params(torch.Generator(device="cuda").manual_seed(1)))
    g = torch.Generator(device="cuda").manual_seed(2)
    coords = torch.rand((N, 7), device="cuda", generator=g)
    dout = (torch.randn((N, 4), device="cuda", generator=g) * 1e-2).half()

    # the same network as torch fp16 modules (cuBLAS GEMMs with the bias in the epilogue, ReLU and concatenations as separate kernels)
    ref = nerf.unpack(P)
    mods = {}
    for name, (W, b) in ref.items():
        lin = torch.nn.Linear(W.shape[1], W.shape[0]).cuda().half()
        with torch.no_grad():
            lin.weight.copy_(W)
            lin.bias.copy_(b)
        mods[name] = lin
    enc = nerf.freq_encode(coords[:, :3], 10).half()
    encd = nerf.freq_encode(coords[:, 4:], 4).half()

    def torch_fwd():
        h = enc
        for i in range(8):
            h = torch.relu(mods[f"pts_linears.{i}"](h))
            if i == 4:
                h = torch.cat([enc, h], -1)
        v = torch.relu(mods["views_linears.0"](torch.cat([mods["feature_linear"](h), encd], -1)))
        return torch.cat([mods["rgb_linear"](v), mods["alpha_linear"](h)], -1)

    state = {}

    def torch_fwd_saved():
        state["y"] = torch_fwd()

    def torch_bwd():
        for m in mods.values():
            m.weight.grad = m.bias.grad = None
        state["y"].backward(dout)

    def ours_fwd_saved():
        state["o"] = ops.nerf_fwd(coords, P, save=True)

    def ours_bwd():
        ops.nerf_bwd(P, state["o"][1], dout)

    # warm-up of every shape, then alternate the two implementations
    for _ in range(3):
        ours_fwd_saved(); ours_bwd(); torch_fwd_saved(); torch_bwd()
    torch.cuda.synchronize()
    t = {k: [] for k in ("ours_fwd", "ours_bwd", "torch_fwd", "torch_bwd", "ours_infer")}
    for _ in range(args.reps):
        t["ours_fwd"] += timed(ours_fwd_saved, 1)
        t["ours_bwd"] += timed(ours_bwd, 1)
        t["torch_fwd"] += timed(torch_fwd_saved, 1)
        t["torch_bwd"] += timed(torch_bwd, 1)
        t["ours_infer"] += timed(lambda: ops.nerf_fwd(coords, P), 1)
    state.clear()
    res = dict(card=card(), rows=N, fwd_mflop_per_row=FWD_FLOP / 1e6, bwd_mflop_per_row=BWD_FLOP / 1e6)
    for k, v in t.items():
        s = stats(v)
        flop = (FWD_FLOP if "fwd" in k or "infer" in k else BWD_FLOP) * N
        s["tflops"] = round(flop / (s["median_ms"] * 1e-3) / 1e12, 1)
        res[k] = s
    res["fwd_bwd_speedup_vs_torch"] = round((res["torch_fwd"]["median_ms"] + res["torch_bwd"]["median_ms"]) /
                                            (res["ours_fwd"]["median_ms"] + res["ours_bwd"]["median_ms"]), 3)

    # training steps of nerf_cfg (synthetic stand-in at 200x200, 20 views) through the Runner's per-operator step
    cfg = get_cfg()
    cfg.dataset.train.n_images, cfg.dataset.train.H, cfg.dataset.train.W = 20, 200, 200
    cfg.dataset.val = None
    r = Runner()
    for _ in range(64):
        r.train_step_autograd()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        r.train_step_autograd()
    torch.cuda.synchronize()
    res["train_step_ms"] = round((time.perf_counter() - t0) * 1e3 / args.steps, 3)
    res["train_rays_per_batch"] = int(r.sampler.n_rays_per_batch)
    res["train_samples_last_step"] = int(r.sampler.n_samples_dev.item())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
