#!/usr/bin/env python
"""What honouring a capture's lens costs on the GPU.

    python tools/lens_bench.py [--reps 200] [--steps 300] [--out FILE]

1. ngp_prepare_batch against ngp_prepare_batch_lens (the fox capture's lens) at 2^12 .. 2^20 rays of 1080x1920 uint8 images: median of
   CUDA-event timings of single launches, the two entry points alternated launch by launch.
2. Training it/s of the fox configuration on its stand-in (fox_cfg, synthetic, 1080x1920 views): images taken through the fox lens and
   trained with undistort=True, against the pinhole stand-in trained as shipped; each runs `--steps` timed steps after 64 warm-up
   steps, pinhole and lens in turn, twice.
The card's name, power limit and SM clock limit are printed beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FOX_LENS = (0.0578421, -0.0805099, -0.000980296, 0.00015575)          # data/fox/transforms_train.json


def gpu_state():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def bench_prepare_batch(reps):
    import torch
    from jnerf_b200 import ops
    n_img, W, H = 8, 1080, 1920
    g = torch.Generator(device="cuda").manual_seed(0)
    xf = torch.eye(3, 4, device="cuda").T.reshape(1, 12).repeat(n_img, 1).contiguous()
    focal = torch.tensor([[1375.52, 1374.49]] * n_img, device="cuda")
    principal = torch.tensor([[554.558 / W, 965.268 / H]] * n_img, device="cuda")
    dist = torch.tensor([FOX_LENS] * n_img, device="cuda")
    images = torch.randint(0, 256, (n_img, H * W, 4), device="cuda", generator=g, dtype=torch.uint8)
    rows = []
    for lg in range(12, 21, 2):
        n = 1 << lg
        pix = torch.randint(0, n_img * H * W, (n,), device="cuda", generator=g, dtype=torch.int32)
        bg = torch.rand((n, 3), device="cuda", generator=g)
        runs = {"pinhole": lambda: ops.prepare_batch(pix, W, H, xf, focal, principal, images, bg),
                "lens": lambda: ops.prepare_batch(pix, W, H, xf, focal, principal, images, bg, distortion=dist)}
        for f in runs.values():
            for _ in range(10):
                f()
        ms = {k: [] for k in runs}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(reps):
            for k, f in runs.items():
                ev[0].record()
                f()
                ev[1].record()
                ev[1].synchronize()
                ms[k].append(ev[0].elapsed_time(ev[1]))
        med = {k: sorted(v)[len(v) // 2] * 1e3 for k, v in ms.items()}
        rows.append({"rays": n, "prepare_batch_us": round(med["pinhole"], 2), "prepare_batch_lens_us": round(med["lens"], 2),
                     "ratio": round(med["lens"] / med["pinhole"], 3)})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def bench_training(steps, rounds=2):
    """Runners share the global configuration, so they are built, timed and dropped one at a time, pinhole and lens in turn."""
    import torch
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    rates = {"pinhole": [], "lens": []}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for name, lens in (("pinhole", None), ("lens", FOX_LENS)):
            get_cfg().clear()
            update_cfg(**fox_cfg(fp16=True, synthetic=True, undistort=lens is not None, seed=1))
            cfg = get_cfg()
            cfg.dataset.train.n_images = 20
            cfg.dataset.test = None
            if lens:
                cfg.dataset.train.distortion = list(lens)
            r = Runner()
            for _ in range(64):                                        # warm-up, past the first occupancy-grid updates
                r.train_step()
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(steps):
                r.train_step()
            ev[1].record()
            ev[1].synchronize()
            rates[name].append(steps / (ev[0].elapsed_time(ev[1]) * 1e-3))
            del r
            torch.cuda.empty_cache()
    out = {"steps": steps, "it_per_s_pinhole": [round(x, 1) for x in rates["pinhole"]], "it_per_s_lens": [round(x, 1) for x in rates["lens"]]}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from jnerf_b200 import lib
    if not torch.cuda.is_available():
        raise SystemExit("lens_bench.py times CUDA kernels and needs a GPU")
    lib.load()
    state = gpu_state()
    print(state, flush=True)
    res = {"gpu": state, "prepare_batch": bench_prepare_batch(args.reps), "training": bench_training(args.steps)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
