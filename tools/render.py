#!/usr/bin/env python
"""Render a trained model on the whole-frame renderer (Runner.render_rays): one view, the camera-path video or the test split.

    python tools/render.py --ckpt CKPT (--config-file CFG | --workload lego|fox) --task pose|video|test [--min-transmittance 1e-4] [--out DIR]
    python tools/render.py --workload lego --train-steps 3000 --task test --compare

--ckpt takes this project's .pt checkpoints or the reference's params.pkl.  Without --ckpt, --train-steps trains the stand-in first
(the configuration of tools/train_psnr.py).  --task pose renders the first training view's pose, video the 80-frame spherical path
(DIR/demo.mp4), test every test view (PNGs in DIR, mean PSNR).  Prints one JSON line: frames, W, H, per-frame ms between CUDA events
recorded before and after each frame (median, min, max; for the whole-frame renderer this includes the host read-back of the alive
count after every round), rounds and mean composited samples per pixel.  --compare also times render_img_nosync and the renderer at
min_transmittance 0 on the same views with the same jitter, the three alternating frame by frame."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def summary(ms):
    return {"median": round(statistics.median(ms), 3), "min": round(min(ms), 3), "max": round(max(ms), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config-file", default="", help="a JNeRF config (projects/ngp/configs/*.py)")
    ap.add_argument("--workload", default="lego", choices=["lego", "fox"], help="the synthetic stand-ins, as in tools/train_psnr.py")
    ap.add_argument("--ckpt", default=None, help=".pt checkpoint of this project or the reference's .pkl")
    ap.add_argument("--train-steps", type=int, default=0, help="without --ckpt: train the stand-in for this many steps first")
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--res", type=int, default=800, help="lego stand-in: frame size (the fox stand-in keeps its 1080x1920 frames)")
    ap.add_argument("--task", default="test", choices=["pose", "video", "test"])
    ap.add_argument("--min-transmittance", type=float, default=1e-4)
    ap.add_argument("--compare", action="store_true", help="also time render_img_nosync and min_transmittance 0, alternating")
    ap.add_argument("--out", default="render_out")
    args = ap.parse_args()
    if args.compare and args.task == "video":
        ap.error("--compare needs --task pose or test (render_img_nosync renders dataset views)")

    import torch
    from jnerf_b200 import lib, plugin  # noqa: F401
    from jnerf_b200.plugin import losses as L
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, init_cfg, update_cfg
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg

    lib.load()
    get_cfg().clear()
    if args.config_file:
        init_cfg(args.config_file)
    elif args.workload == "fox":
        update_cfg(**fox_cfg(fp16=True, synthetic=True, seed=1))
        get_cfg().dataset.val = None
    else:
        update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=1))
        cfg = get_cfg()
        for split in ("train", "val", "test"):
            d = cfg.dataset[split]
            d.n_images = args.images
            d.H = d.W = args.res
            d.pop("root_dir", None)
    get_cfg().log_dir, get_cfg().exp_name = os.path.dirname(os.path.abspath(args.out)), os.path.basename(os.path.abspath(args.out))
    runner = Runner()
    if args.ckpt:
        runner.load_ckpt(args.ckpt)
    elif args.train_steps:
        for _ in range(args.train_steps):
            runner.train_step()
    torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    s, eps = runner.sampler, args.min_transmittance
    t0 = time.perf_counter()
    row = {"task": args.task, "min_transmittance": eps}

    if args.task == "video":
        ms, rounds, spp = [], [], []
        real = runner.render_rays

        def timed(o, d, m):                                          # per frame: raygen + every round, CUDA events
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = real(o, d, m)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
            rounds.append(out[3])
            spp.append(float(out[2].float().mean()))
            return out
        runner.render_rays = timed
        path = runner.render(save_path=os.path.join(args.out, "demo.mp4"), min_transmittance=eps)
        W, H = runner.dataset["train"].resolution
        row.update(frames=len(ms), W=W, H=H, ms=summary(ms), rounds=round(statistics.mean(rounds), 2), spp=round(statistics.mean(spp), 3),
                   out=os.path.abspath(path))
    else:
        if args.task == "test":
            if runner.dataset["test"] is None:
                runner.dataset["test"] = build_from_cfg(runner.cfg.dataset.test, DATASETS)
            mode, ds = "test", runner.dataset["test"]
            views = list(range(ds.n_images))
        else:
            mode, ds = "train", runner.dataset["train"]
            views = [0]
        W, H = ds.resolution
        bgc = torch.tensor(runner.background_color, dtype=torch.float32, device="cuda")
        variants = [("new", eps)] + ([("eps0", 0.0), ("nosync", None)] if args.compare else [])
        res = {k: dict(ms=[], rounds=[], spp=[], psnr=[]) for k, _ in variants}

        def run(kind, m, i):
            if kind == "nosync":
                img, tar = runner.render_img_nosync(mode, i)
                return img, tar, None
            if mode == "train":
                o, d = runner.pose_rays(ds.poses[i])
            else:
                o, d = ds.generate_rays_total_test(i)
            img, _, n, rounds = runner._render_frame(o, d, W, H, m)
            tar = ds.rgba_for(torch.arange(H * W, device="cuda", dtype=torch.int32) + i * H * W)
            tar = (tar[:, :3] * tar[:, 3:] + bgc * (1 - tar[:, 3:])).reshape(H, W, 3)
            return img, tar, (n, rounds)

        rng0 = s.rng.copy()
        for kind, m in variants:                                     # warm-up: modules, allocations
            s.rng[:] = rng0
            run(kind, m, views[0])
        torch.cuda.synchronize()
        for i in views:
            for kind, m in variants:                                 # alternating, same jitter for all three
                s.rng[:] = rng0
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                img, tar, extra = run(kind, m, i)
                b.record()
                b.synchronize()
                r = res[kind]
                r["ms"].append(a.elapsed_time(b))
                r["psnr"].append(float(L.mse2psnr(L.img2mse(img, tar)).item()))
                if extra is not None:
                    r["spp"].append(float(extra[0].float().mean()))
                    r["rounds"].append(extra[1])
                if kind == "new" and args.task == "test":
                    runner.save_img(os.path.join(args.out, f"{runner.cfg.exp_name}_r_{i}.png"), img)
                    runner.save_img(os.path.join(args.out, f"{runner.cfg.exp_name}_gt_{i}.png"), tar)
                elif kind == "new":
                    runner.save_img(os.path.join(args.out, "pose.png"), img)
            rng0 = s.rng.copy()
        new = res["new"]
        row.update(frames=len(views), W=W, H=H, ms=summary(new["ms"]), rounds=round(statistics.mean(new["rounds"]), 2),
                   spp=round(statistics.mean(new["spp"]), 3), psnr=round(statistics.mean(new["psnr"]), 3))
        if args.compare:
            e0, ns = res["eps0"], res["nosync"]
            row["compare"] = {"eps0": dict(ms=summary(e0["ms"]), rounds=round(statistics.mean(e0["rounds"]), 2),
                                           spp=round(statistics.mean(e0["spp"]), 3), psnr=round(statistics.mean(e0["psnr"]), 3)),
                              "render_img_nosync": dict(ms=summary(ns["ms"]), psnr=round(statistics.mean(ns["psnr"]), 3))}
    row.update(wall_s=round(time.perf_counter() - t0, 3), gpu=torch.cuda.get_device_name(0), timeout_flag=int(lib.load().ngp_debug_timeout_flag()))
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
