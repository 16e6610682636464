#!/usr/bin/env python
"""Render a trained model on the whole-frame renderer (Runner.render_rays): one view, the camera-path video or the test split.

    python tools/render.py --ckpt CKPT (--config-file CFG | --workload lego|fox|llff) --task pose|video|test [--min-transmittance 1e-4] [--out DIR]
    python tools/render.py --workload lego --train-steps 3000 --task test --compare
    python tools/render.py --workload llff --train-steps 2000 --task video --path spiral --depth

--ckpt takes this project's .pt checkpoints or the reference's params.pkl.  Without --ckpt, --train-steps trains the stand-in first
(the configuration of tools/train_psnr.py).  --task pose renders the first training view's pose, video the 80-frame spherical path
(DIR/demo.mp4), test every test view (PNGs in DIR, mean PSNR).  Prints one JSON line: frames, W, H, per-frame ms between CUDA events
recorded before and after each frame (median, min, max; for the whole-frame renderer this includes the host read-back of the alive
count after every round), rounds and mean composited samples per pixel.  --compare also times render_img_nosync and the renderer at
min_transmittance 0 on the same views with the same jitter, the three alternating frame by frame.  --depth also renders depth maps:
the video gains DIR/demo_depth.mp4 and its timing is of the depth renders; pose and test render every view with and without depth,
alternating, write the depth maps ({exp}_depth_{i}.npy / .png, pose_depth.*) and add the depth-on timing to the JSON line.  --path
spiral flies the spiral of a forward-facing capture (utils/camera_path.path_spiral) instead of the spherical path; it needs a dataset
with near / far bounds (LLFF).  --workload llff is the forward-facing stand-in of tools/train_psnr.py, written to a temporary directory.
--normals also renders normal maps (fused NGP models only), as --depth does depth maps: the video gains DIR/demo_normal.mp4, pose and
test render every view with and without normals, alternating, and write {exp}_normal_{i}.npy / .png (pose_normal.*); the JSON line
gains the normal-on timing and, for pose and test, ngp_density_grad alone against the fused forward (ngp_network_fwd) on the same
march rows of the first view, in rows per second."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def summary(ms):
    return {"median": round(statistics.median(ms), 3), "min": round(min(ms), 3), "max": round(max(ms), 3)}


def density_grad_rate(runner, ds, i, mode, reps=20):
    """ngp_density_grad and ngp_network_fwd over the same rows, the march samples of view i (ray-ordered, as a render round holds them):
    rows and median ms of each over `reps` alternating launches (CUDA events), and rows per second."""
    import torch
    from jnerf_b200 import ops
    s, m = runner.sampler, runner.model
    o, d = runner.pose_rays(ds.poses[i]) if mode == "train" else ds.generate_rays_total_test(i)
    rng = s.rng.copy()
    coords, _, _, counters = ops.march(o.contiguous(), d.contiguous(), s.density_grid_bitfield, s.aabb_range, 1 << 23, s.cone_angle_constant,
                                       s.near_distance, s.NERF_CASCADES, s.const_dt, rng)
    rows = coords[:int(counters[1].item())].contiguous()                      # the compacted samples, at most the buffer's 2^23
    n = rows.shape[0]
    grid, lv, wd, wr = m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights
    out = torch.empty((n, 4), dtype=torch.float16, device="cuda")
    grad = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    kernels = {"density_grad": lambda: ops.density_grad(rows, grid, lv, wd, out=grad),
               "network_fwd": lambda: ops.network_fwd(rows, grid, lv, wd, wr, save_enc=False, out=out)}
    ms = {k: [] for k in kernels}
    for f in kernels.values():
        f()
    for _ in range(reps):
        for k, f in kernels.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {"rows": n, **{k: dict(ms=round(statistics.median(v), 4), rows_per_s=round(n / statistics.median(v) * 1e3, 1)) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config-file", default="", help="a JNeRF config (projects/ngp/configs/*.py)")
    ap.add_argument("--workload", default="lego", choices=["lego", "fox", "llff"], help="the synthetic stand-ins, as in tools/train_psnr.py")
    ap.add_argument("--ckpt", default=None, help=".pt checkpoint of this project or the reference's .pkl")
    ap.add_argument("--train-steps", type=int, default=0, help="without --ckpt: train the stand-in for this many steps first")
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--res", type=int, default=800, help="lego stand-in: frame size (the fox stand-in keeps its 1080x1920 frames)")
    ap.add_argument("--task", default="test", choices=["pose", "video", "test"])
    ap.add_argument("--min-transmittance", type=float, default=1e-4)
    ap.add_argument("--compare", action="store_true", help="also time render_img_nosync and min_transmittance 0, alternating")
    ap.add_argument("--depth", action="store_true", help="also render depth maps (and time them)")
    ap.add_argument("--normals", action="store_true", help="also render normal maps (and time them and the density-gradient kernel)")
    ap.add_argument("--path", default="spherical", choices=["spherical", "spiral"], help="camera path of --task video")
    ap.add_argument("--out", default="render_out")
    args = ap.parse_args()
    if args.compare and args.task == "video":
        ap.error("--compare needs --task pose or test (render_img_nosync renders dataset views)")
    if args.path != "spherical" and args.task != "video":
        ap.error("--path is the camera path of --task video")

    import torch
    from jnerf_b200 import lib, plugin  # noqa: F401
    from jnerf_b200.plugin import losses as L
    from jnerf_b200.runner import Runner, fox_cfg, image_resolution, lego_cfg, llff_cfg
    from jnerf_b200.utils.config import get_cfg, init_cfg, update_cfg
    from jnerf_b200.utils.registry import DATASETS, build_from_cfg

    lib.load()
    get_cfg().clear()
    tmp = None
    if args.config_file:
        init_cfg(args.config_file)
    elif args.workload == "llff":
        import tempfile
        from jnerf_b200.plugin.dataset import write_synthetic_llff
        tmp = tempfile.TemporaryDirectory()
        write_synthetic_llff(tmp.name, n_images=args.images if args.images != 100 else 20, H=8 * 192, W=8 * 256)   # read at 192 x 256
        update_cfg(**llff_cfg(tmp.name, fp16=True, seed=1))
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
        poses = None
        if args.path == "spiral":
            from jnerf_b200.utils.camera_path import path_spiral
            tr = runner.dataset["train"]
            if getattr(tr, "bounds", None) is None:
                sys.exit(f"--path spiral needs a forward-facing capture with near / far bounds (LLFFDataset); {type(tr).__name__} has none")
            poses = path_spiral(tr.poses, tr.bounds)

        def timed(o, d, m, **kw):                                    # per frame: raygen + every round, CUDA events
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = real(o, d, m, **kw)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
            rounds.append(out[3])
            spp.append(float(out[2].float().mean()))
            return out
        runner.render_rays = timed
        path = runner.render(save_path=os.path.join(args.out, "demo.mp4"), min_transmittance=eps, depth=args.depth, poses=poses,
                              normals=args.normals)
        W, H = runner.dataset["train"].resolution
        row.update(frames=len(ms), W=W, H=H, ms=summary(ms), rounds=round(statistics.mean(rounds), 2), spp=round(statistics.mean(spp), 3),
                   out=os.path.abspath(path), path=args.path, depth=args.depth,
                   normals=args.normals)
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
        variants = [("new", eps)] + ([("depth", eps)] if args.depth else []) + ([("normal", eps)] if args.normals else []) + ([("eps0", 0.0), ("nosync", None)] if args.compare else [])
        res = {k: dict(ms=[], rounds=[], spp=[], psnr=[]) for k, _ in variants}

        def run(kind, m, i):
            if kind == "nosync":
                img, tar = runner.render_img_nosync(mode, i)
                return img, tar, None
            if mode == "train":
                o, d = runner.pose_rays(ds.poses[i])
                W, H = ds.resolution
            else:
                o, d = ds.generate_rays_total_test(i)
                W, H = image_resolution(ds, i)                       # every test view at its own size
            if kind == "depth":
                img, alpha, n, rounds, dep = runner._render_frame(o, d, W, H, m, depth_scale=float(ds.scale))
            elif kind == "normal":
                img, alpha, n, rounds, dep = runner._render_frame(o, d, W, H, m, normals=True)     # dep: the normal map
            else:
                img, alpha, n, rounds = runner._render_frame(o, d, W, H, m)
                dep = None
            pix = ds.image_pixels(i) if hasattr(ds, "image_pixels") else torch.arange(H * W, device="cuda", dtype=torch.int32) + i * H * W
            tar = ds.rgba_for(pix)
            tar = (tar[:, :3] * tar[:, 3:] + bgc * (1 - tar[:, 3:])).reshape(H, W, 3)
            return img, tar, (n, rounds, dep, alpha)

        if args.depth or args.normals:
            from PIL import Image
            from jnerf_b200.runner import depth_to_grey, normal_to_rgb
        if args.depth:
            near, far = runner.depth_range([ds.poses[i] for i in views], ds)
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
                elif kind == "depth":
                    stem = os.path.join(args.out, f"{runner.cfg.exp_name}_depth_{i}" if args.task == "test" else "pose_depth")
                    np.save(stem + ".npy", extra[2].cpu().numpy())
                    Image.fromarray(depth_to_grey(extra[2], extra[3], near, far), "L").save(stem + ".png")
                elif kind == "normal":
                    stem = os.path.join(args.out, f"{runner.cfg.exp_name}_normal_{i}" if args.task == "test" else "pose_normal")
                    np.save(stem + ".npy", extra[2].cpu().numpy())
                    Image.fromarray(normal_to_rgb(extra[2], extra[3]), "RGB").save(stem + ".png")
            rng0 = s.rng.copy()
        new = res["new"]
        row.update(frames=len(views), W=W, H=H, ms=summary(new["ms"]), rounds=round(statistics.mean(new["rounds"]), 2),
                   spp=round(statistics.mean(new["spp"]), 3), psnr=round(statistics.mean(new["psnr"]), 3))
        if args.depth:
            dp = res["depth"]
            over = [x - y for x, y in zip(dp["ms"], new["ms"])]
            row["depth"] = dict(ms=summary(dp["ms"]), overhead_ms=summary(over), psnr=round(statistics.mean(dp["psnr"]), 3),
                                near_far=[round(near, 4), round(far, 4)])
        if args.normals:
            nm = res["normal"]
            over = [x - y for x, y in zip(nm["ms"], new["ms"])]
            row["normals"] = dict(ms=summary(nm["ms"]), overhead_ms=summary(over), psnr=round(statistics.mean(nm["psnr"]), 3),
                                  kernel=density_grad_rate(runner, ds, views[0], mode))
        if args.compare:
            e0, ns = res["eps0"], res["nosync"]
            row["compare"] = {"eps0": dict(ms=summary(e0["ms"]), rounds=round(statistics.mean(e0["rounds"]), 2),
                                           spp=round(statistics.mean(e0["spp"]), 3), psnr=round(statistics.mean(e0["psnr"]), 3)),
                              "render_img_nosync": dict(ms=summary(ns["ms"]), psnr=round(statistics.mean(ns["psnr"]), 3))}
    row.update(wall_s=round(time.perf_counter() - t0, 3), gpu=torch.cuda.get_device_name(0), timeout_flag=int(lib.load().ngp_debug_timeout_flag()))
    print(json.dumps(row), flush=True)
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
