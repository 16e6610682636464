#!/usr/bin/env python
"""Train the lego configuration on the synthetic stand-in scene and report held-out PSNR against steps and device time.

    python tools/train_psnr.py [--steps 5000] [--images 100] [--res 400] [--evals 500,1000,2000,5000] [--out gpurun_out/psnr.json]
    python tools/train_psnr.py --workload llff [--data-dir CAPTURE] [--images 40]
    python tools/train_psnr.py --workload fox [--data-dir CAPTURE] [--undistort] [--distortion K1 K2 P1 P2]
    python tools/train_psnr.py --workload frames [--data-dir CAPTURE] [--res 400] [--images 100]

This is the quality check that goes with bench.py's throughput number: same Runner.train_step path, same configuration
(projects/ngp/configs/ngp_base.py + fp16), validation views drawn from cameras the model never trains on
(runner.py:86-99 val_img semantics: mean over images of -10 log10 MSE against the alpha-composited target)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5000)
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--res", type=int, default=400)
    ap.add_argument("--evals", default="250,500,1000,2000,3500,5000")
    ap.add_argument("--val-images", type=int, default=4)
    ap.add_argument("--out", default=None)
    ap.add_argument("--budget-seconds", type=float, default=0.0,
                    help="BASELINE metric 'PSNR@5min': keep training after --steps until this much device time has been spent on training "
                         "steps or the configuration's tot_train_steps (40 000, ngp_base.py) is reached, then evaluate once more")
    ap.add_argument("--data-dir", default=None, help="a real capture in the reference's dataset layout (train/val splits) instead of the stand-in")
    ap.add_argument("--workload", default="lego", choices=["lego", "fox", "llff", "frames"],
                    help="fox = projects/ngp/configs/ngp_fox.py (aabb_scale from the capture, cone stepping); PSNR on training views (the capture has no val split). "
                         "llff = projects/ngp/configs/ngp_llff.py (aabb_scale 64: 7 occupancy cascades, every 8th view held out) on --data-dir, an LLFF "
                         "capture (poses_bounds.npy + images/), or on the forward-facing stand-in written to a temporary directory. "
                         "frames = ngp_base.py on a capture whose frames carry their own cameras (NerfDataset(per_frame_cameras=True)): --data-dir, or "
                         "the lego stand-in written to a temporary directory with frames cycling through a res x res camera, a 1.2 res x 0.8 res one "
                         "and a zoomed 0.8 res x 1.2 res one with an off-centre principal point; PSNR on the test split")
    ap.add_argument("--undistort", action="store_true", help="fox: train and evaluate through the capture's lens (datasets' undistort=True)")
    ap.add_argument("--distortion", type=float, nargs=4, default=None, metavar=("K1", "K2", "P1", "P2"),
                    help="fox stand-in: take its images through this lens (k1 k2 p1 p2)")
    args = ap.parse_args()
    if (args.undistort or args.distortion) and args.workload != "fox":
        ap.error("--undistort and --distortion go with --workload fox")
    if args.distortion and args.data_dir:
        ap.error("--distortion is the stand-in's lens; a capture brings its own in its transforms json")

    import torch
    from jnerf_b200 import lib, plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg, llff_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg

    lib.load()
    get_cfg().clear()
    tmp = None
    if args.workload == "llff":
        root = args.data_dir
        if root is None:
            import tempfile
            from jnerf_b200.plugin.dataset import write_synthetic_llff
            tmp = tempfile.TemporaryDirectory()
            root = tmp.name
            write_synthetic_llff(root, n_images=args.images, H=8 * 192, W=8 * 256)    # read at 192 x 256 (factor 8); the fern capture is read at 378 x 504
        update_cfg(**llff_cfg(root, fp16=True, seed=1))
        cfg = get_cfg()
    elif args.workload == "frames":
        root = args.data_dir
        if root is None:
            import tempfile
            from jnerf_b200.plugin.dataset import write_synthetic_frames
            tmp = tempfile.TemporaryDirectory()
            root = tmp.name
            r = args.res
            f = 0.5 * r / 0.36                                          # the stand-in's field of view (camera_angle_x 0.6911)
            cams = [(r, r, f, f, r / 2, r / 2), (int(1.2 * r), int(0.8 * r), f, f, 0.6 * r, 0.4 * r),
                    (int(0.8 * r), int(1.2 * r), 1.5 * f, 1.5 * f, 0.28 * r, 0.75 * r)]
            write_synthetic_frames(root, cams, n_images=args.images)
        update_cfg(**lego_cfg(fp16=True, synthetic=False, seed=1))
        cfg = get_cfg()
        for split in ("train", "val", "test"):
            cfg.dataset[split].update(root_dir=root, per_frame_cameras=True, mode="test" if split == "val" else split)
        cfg.dataset.test = None
    elif args.workload == "fox":
        update_cfg(**fox_cfg(fp16=True, synthetic=args.data_dir is None, undistort=args.undistort, seed=1))
        cfg = get_cfg()
        if args.distortion:
            cfg.dataset.train.distortion = cfg.dataset.test.distortion = list(args.distortion)
        if args.data_dir:
            cfg.dataset.train.root_dir = args.data_dir
            cfg.dataset.test.root_dir = args.data_dir
        cfg.dataset.val = None                                      # Runner evaluates on the training views then
    else:
        update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=1))
        cfg = get_cfg()
        for split in ("train", "val"):
            d = cfg.dataset[split]
            d.n_images = args.images
            d.H = d.W = args.res
            d.pop("root_dir", None)
        cfg.dataset.test = None
        if args.data_dir:
            for split in ("train", "val"):
                cfg.dataset[split] = dict(type="NerfDataset", root_dir=args.data_dir, batch_size=4096, mode=split, preload_shuffle=split == "train")
    runner = Runner()
    evals = sorted({int(x) for x in args.evals.split(",") if int(x) <= args.steps} | {args.steps})
    rows, train_ms, done = [], 0.0, 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for target in evals:
        torch.cuda.synchronize()
        e0.record()
        rays = 0
        for _ in range(target - done):
            rays += runner.sampler.n_rays_per_batch
            runner.train_step()
        e1.record()
        torch.cuda.synchronize()
        train_ms += e0.elapsed_time(e1)
        done = target
        psnr = runner.psnr("val", max_images=args.val_images)
        row = {"step": done, "train_seconds": round(train_ms * 1e-3, 3), "val_psnr_db": round(psnr, 3), "loss": float(runner.last_loss.float().mean().item()),
               "rays_per_batch": int(runner.sampler.n_rays_per_batch)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    res = {"config": f"ngp_base + fp16, {args.images} synthetic {args.res}x{args.res} views, {args.val_images} held-out views", "curve": rows}
    if args.data_dir:
        res["config"] = f"ngp_base + fp16 on {args.data_dir}, {args.val_images} validation views"
    if args.workload == "fox":
        res["config"] = (f"ngp_fox.py (fp16, cone stepping) on {args.data_dir or 'the synthetic fox stand-in'}, PSNR on {args.val_images} training views "
                         f"(the capture has no validation split)" + (f", images through the lens {args.distortion}" if args.distortion else "")
                         + (", rays undistorted" if args.undistort else ""))
    if args.workload == "frames":
        res["config"] = (f"ngp_base + fp16 on {args.data_dir or 'the per-frame-camera lego stand-in'}, per_frame_cameras=True: "
                         f"{runner.dataset['train'].n_images} training views of {sorted({runner.dataset['train'].image_resolution(i) for i in range(runner.dataset['train'].n_images)})}, "
                         f"PSNR on {args.val_images} held-out views")
    if args.workload == "llff":
        res["config"] = (f"ngp_llff.py (fp16, cone stepping, aabb_scale 64) on {args.data_dir or 'the forward-facing stand-in'}: "
                         f"{runner.dataset['train'].n_images} training views of {runner.W}x{runner.H}, PSNR on {args.val_images} held-out views")
    if args.budget_seconds > 0:
        tot = int(cfg.tot_train_steps or 40000)
        while train_ms * 1e-3 < args.budget_seconds and done < tot:
            n = min(1000, tot - done)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(n):
                runner.train_step()
            e1.record()
            torch.cuda.synchronize()
            train_ms += e0.elapsed_time(e1)
            done += n
        psnr = runner.psnr("val", max_images=args.val_images)
        res["psnr_at_budget"] = {"budget_seconds": args.budget_seconds, "steps": done, "train_seconds": round(train_ms * 1e-3, 3),
                                 "val_psnr_db": round(psnr, 3), "stopped_by": "tot_train_steps" if done >= tot else "budget"}
        print(json.dumps(res["psnr_at_budget"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
