#!/usr/bin/env python
"""Export a trained model as a coloured mesh: the reference's tools/extract_mesh.py on the device (Runner.extract_mesh).

    python tools/extract_mesh.py --ckpt CKPT (--config-file CFG | --workload lego|fox) [--resolution 512] [--mcube_smooth] [--out DIR]
    python tools/extract_mesh.py --workload lego --train-steps 3000 [--resolution 512] [--mcube_smooth] [--out DIR]

--ckpt takes this project's .pt checkpoints or the reference's params.pkl.  Without --ckpt, --train-steps trains the stand-in first
(the configuration of tools/train_psnr.py).  Writes DIR/mesh-origin.ply and DIR/mesh-color.ply and prints one JSON line: vertex and
triangle counts before and after the component filter and the device time of every stage (CUDA events); with --mcube_smooth also
the smoothing method, its iterations and its band variables."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config-file", default="", help="a JNeRF config (projects/ngp/configs/*.py)")
    ap.add_argument("--workload", default="lego", choices=["lego", "fox"], help="the synthetic stand-ins, as in tools/train_psnr.py")
    ap.add_argument("--ckpt", default=None, help=".pt checkpoint of this project or the reference's .pkl")
    ap.add_argument("--train-steps", type=int, default=0, help="without --ckpt: train the stand-in for this many steps first")
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--res", type=int, default=400)
    ap.add_argument("--resolution", type=int, default=512, help="lattice points per axis, in [2, 1024]")
    ap.add_argument("--out", default="mesh_out")
    ap.add_argument("--mcube_smooth", action="store_true",
                    help="smooth the lattice (constrained up to 512^3, Gaussian above) and march it at 0: no terraces from the integer density")
    args = ap.parse_args()
    if not 2 <= args.resolution <= 1024:
        ap.error("--resolution must be in [2, 1024]")

    import torch
    from jnerf_b200 import lib, plugin  # noqa: F401
    from jnerf_b200.runner import Runner, fox_cfg, lego_cfg
    from jnerf_b200.utils.config import get_cfg, init_cfg, update_cfg

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
        for split in ("train", "val"):
            d = cfg.dataset[split]
            d.n_images = args.images
            d.H = d.W = args.res
            d.pop("root_dir", None)
        cfg.dataset.test = None
    runner = Runner()
    if args.ckpt:
        runner.load_ckpt(args.ckpt)
    elif args.train_steps:
        for _ in range(args.train_steps):
            runner.train_step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = runner.extract_mesh(args.out, resolution=args.resolution, mcube_smooth=args.mcube_smooth)
    wall = time.perf_counter() - t0
    row = {"resolution": args.resolution, "vertices_origin": res["n_verts_origin"], "triangles_origin": res["n_tris_origin"],
           "vertices": res["n_verts"], "triangles": res["n_tris"], "stage_ms": res["stage_ms"],
           "device_ms_total": round(sum(res["stage_ms"].values()), 3), "wall_s": round(wall, 3), "gpu": torch.cuda.get_device_name(0),
           "out": os.path.abspath(args.out)}
    if args.mcube_smooth:
        sm = res["smooth"]
        row.update(smooth_method=sm["method"], smooth_iters=sm["iterations"], band_variables=sm["band_variables"])
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
