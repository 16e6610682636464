#!/usr/bin/env python
"""What training on a capture whose frames carry their own cameras costs on the GPU.

    python tools/frame_cameras_bench.py [--reps 200] [--steps 300] [--out FILE]

1. The batch kernel at 2^12 .. 2^20 rays of uint8 images, median of CUDA-event timings of single launches, the entry points alternated
   launch by launch:
   - one same-size capture (8 frames of 1080x1920): ngp_prepare_batch against ngp_prepare_batch_cams on the same pixels, so the
     difference is the cost of the search over the pixel offsets;
   - a mixed capture of about the same pixel count (8 frames: 1080x1920, 1920x1080 and a zoomed 1080x1920 with an off-centre principal
     point, in turn): ngp_prepare_batch_cams;
   - the same two with 256 frames of 300x400 (and 400x300 in the mixed one), where the search takes 8 steps instead of 3.
2. Training it/s of the lego configuration on its stand-in with 40 views: frames cycling through an 800x800 camera, a 960x640 one and a
   zoomed 640x960 one with an off-centre principal point (per-frame cameras, the `_cams` entry points), against all 40 frames with the
   800x800 camera (the existing entry points); each runs `--steps` timed steps after 64 warm-up steps, in turn, twice.
The card's name, power limit and SM clock limit are printed beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_state():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def tables(cams):
    import numpy as np
    import torch
    wh = np.array([c[:2] for c in cams], np.int64)
    offsets = np.concatenate([[0], np.cumsum(wh[:, 0] * wh[:, 1])])
    n = len(cams)
    return dict(offsets=torch.from_numpy(offsets.astype(np.int32)).cuda(), wh=torch.from_numpy(wh.astype(np.int32)).cuda(),
                xf=torch.eye(3, 4, device="cuda").T.reshape(1, 12).repeat(n, 1).contiguous(),
                focal=torch.tensor([c[2:4] for c in cams], dtype=torch.float32, device="cuda"),
                principal=torch.tensor([[c[4] / c[0], c[5] / c[1]] for c in cams], dtype=torch.float32, device="cuda"), total=int(offsets[-1]))


def bench_prepare_batch(reps):
    import torch
    from jnerf_b200 import ops
    fox = (1080, 1920, 1375.52, 1374.49, 554.558, 965.268)
    captures = {
        8: ([fox] * 8, [fox, (1920, 1080, 1375.52, 1374.49, 965.268, 554.558), (1080, 1920, 2751.0, 2749.0, 300.0, 1300.0)] * 2 + [fox] * 2),
        256: ([(300, 400, 350.0, 350.0, 150.0, 200.0)] * 256, [(300, 400, 350.0, 350.0, 150.0, 200.0), (400, 300, 350.0, 350.0, 200.0, 150.0)] * 128),
    }
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for n_img, (same_cams, mixed_cams) in captures.items():
        same, mixed = tables(same_cams), tables(mixed_cams)
        W, H = same_cams[0][:2]
        img_same = torch.randint(0, 256, (same["total"], 4), device="cuda", generator=g, dtype=torch.uint8)
        img_mixed = torch.randint(0, 256, (mixed["total"], 4), device="cuda", generator=g, dtype=torch.uint8)
        for lg in range(12, 21, 2):
            n = 1 << lg
            pix_s = torch.randint(0, same["total"], (n,), device="cuda", generator=g, dtype=torch.int32)
            pix_m = torch.randint(0, mixed["total"], (n,), device="cuda", generator=g, dtype=torch.int32)
            bg = torch.rand((n, 3), device="cuda", generator=g)
            s, m = same, mixed
            runs = {"prepare_batch": lambda: ops.prepare_batch(pix_s, W, H, s["xf"], s["focal"], s["principal"], img_same, bg),
                    "cams_same": lambda: ops.prepare_batch_cams(pix_s, s["offsets"], s["wh"], s["xf"], s["focal"], s["principal"], img_same, bg),
                    "cams_mixed": lambda: ops.prepare_batch_cams(pix_m, m["offsets"], m["wh"], m["xf"], m["focal"], m["principal"], img_mixed, bg)}
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
            rows.append({"frames": n_img, "rays": n, "prepare_batch_us": round(med["prepare_batch"], 2),
                         "prepare_batch_cams_same_us": round(med["cams_same"], 2), "prepare_batch_cams_mixed_us": round(med["cams_mixed"], 2),
                         "ratio_same": round(med["cams_same"] / med["prepare_batch"], 3), "ratio_mixed": round(med["cams_mixed"] / med["prepare_batch"], 3)})
            print(json.dumps(rows[-1]), flush=True)
    return rows


STAND_IN = {"one": [(800, 800, 1111.1, 1111.1, 400.0, 400.0)],
            "mixed": [(800, 800, 1111.1, 1111.1, 400.0, 400.0), (960, 640, 1111.1, 1111.1, 480.0, 320.0),
                      (640, 960, 1666.7, 1666.7, 224.0, 720.0)]}


def bench_training(steps, rounds=2):
    """Runners share the global configuration, so they are built, timed and dropped one at a time, one camera and mixed in turn."""
    import torch
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    rates = {k: [] for k in STAND_IN}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for name, cams in STAND_IN.items():
            get_cfg().clear()
            update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=1))
            cfg = get_cfg()
            cfg.dataset.train.n_images = 40
            cfg.dataset.train.cameras = cams
            cfg.dataset.val = cfg.dataset.test = None
            r = Runner()
            assert r.dataset["train"].frame_cameras == (name == "mixed")
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
    out = {"steps": steps, "it_per_s_one_camera": [round(x, 1) for x in rates["one"]], "it_per_s_mixed": [round(x, 1) for x in rates["mixed"]]}
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
        raise SystemExit("frame_cameras_bench.py times CUDA kernels and needs a GPU")
    lib.load()
    state = gpu_state()
    print(state, flush=True)
    res = {"gpu": state, "prepare_batch": bench_prepare_batch(args.reps), "training": bench_training(args.steps)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
