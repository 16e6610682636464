#!/usr/bin/env python
"""Plenoxels training step on the GPU: Svox2Runner on the procedural stand-in (SyntheticSvoxDataset), 5000 rays a step, at 256^3 and at
512^3 after a resample.  Per step, from CUDA events: the fused train step (ray generation, forward, MSE gradient, backward), the two sparse
TV launches, the RMSprop sweep, and the whole step (events recorded by Svox2Runner.train_step itself).  Where the reference's kernels are
built (oracle/svox.mk), its forward and backward kernels run on one 5000-ray batch of the same grid between our steps, alternating.  Each resolution is first trained for --warmup steps, so that the timed steps march
a grid that has started to fit the scene.  Prints one JSON line with the GPU's name and power limit, read in the same run.

    python tools/svox2_bench.py [--steps 50] [--warmup 200] [--images 20] [--size 400]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jnerf_b200 import plugin  # noqa: E402,F401
from jnerf_b200.svox2_runner import Svox2Runner, svox2_cfg  # noqa: E402
from jnerf_b200.utils.config import get_cfg, update_cfg  # noqa: E402


def ref_kernels():
    """The reference's own forward / backward kernels (oracle/_ref/libref_svox.so, oracle/svox.mk), or None where they are not built."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import svox_cpu_backend
    return svox_cpu_backend


def measure(r, steps, warmup, gstep0, ref=None):
    """Mean per-step stage times of Svox2Runner.train_step; with ref, the reference's render + backward kernels on one batch of the
    same grid, launched between our steps (alternating), with their float gradients into buffers of their own."""
    for i in range(warmup):
        r.train_step(gstep0 + i)
    torch.cuda.synchronize()
    lib = ref.ref_svox_lib() if ref is not None else None
    if lib is not None:
        ds, g = r.dataset["train"], r.model
        pix = torch.randint(0, ds.n_rays, (r.cfg.batch_size,), generator=torch.Generator().manual_seed(0)).numpy()
        o, d = ref.pixel_rays_f32(pix, ds.w, ds.h, ds.c2w_rows.cpu().numpy(), (ds.focal, ds.focal, ds.w * 0.5, ds.h * 0.5))
        o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
        gt = torch.rand((len(pix), 3), device="cuda")
        xf = torch.from_numpy(g.xform()).cuda()
        rgb = torch.empty((len(pix), 3), device="cuda")
        gd, gs = torch.zeros(g.capacity, device="cuda"), torch.zeros((g.capacity, 27), device="cuda")
        X, Y, Z = g._links.shape
        args = [o.data_ptr(), d.data_ptr(), g._links.data_ptr(), X, Y, Z, g.capacity, g.density_data.data_ptr(), g.sh_data.data_ptr(),
                xf[:3].data_ptr(), xf[3:].data_ptr()]
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(6)] for _ in range(steps)]
    for i, ev in enumerate(evs):
        r.train_step(gstep0 + warmup + i, events=ev)
        if lib is not None:
            assert lib.ref_svox_render(len(pix), *args, rgb.data_ptr(), None) == 0
            ev[4].record()
            assert lib.ref_svox_backward(len(pix), *args, gt.data_ptr(), rgb.data_ptr(), gd.data_ptr(), gs.data_ptr(), None) == 0
            ev[5].record()
    torch.cuda.synchronize()
    r.optimizer.check_overflow()
    ms = lambda a, b: round(sum(ev[a].elapsed_time(ev[b]) for ev in evs) / steps, 4)  # noqa: E731
    res = {"train_step_ms": ms(0, 1), "tv_ms": ms(1, 2), "rmsprop_ms": ms(2, 3), "total_ms": ms(0, 3), "capacity": int(r.model.capacity)}
    if lib is not None:
        res.update(ref_forward_ms=ms(3, 4), ref_backward_ms=ms(4, 5), ref_fwd_bwd_ms=ms(3, 5))
        res["train_step_speedup_vs_ref_fwd_bwd"] = round(res["ref_fwd_bwd_ms"] / res["train_step_ms"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--images", type=int, default=20)
    ap.add_argument("--size", type=int, default=400)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "svox2_bench.py measures on the GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    get_cfg().clear()
    c = svox2_cfg(synthetic=True, log_dir=tempfile.mkdtemp())
    for s in ("train", "test"):
        c["dataset"][s].update(n_images=a.images, H=a.size, W=a.size)
    update_cfg(**c)
    r = Svox2Runner()
    r.model.param_init(r.cfg)
    res = {"gpu": smi.strip(), "rays": r.cfg.batch_size, "images": a.images, "image_size": a.size}
    ref = ref_kernels()
    res["reference_kernels"] = "built" if ref.ref_svox_lib() is not None else "not measured (oracle/_ref/libref_svox.so is not built)"
    res["reso_256"] = measure(r, a.steps, a.warmup, 0, ref)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    r.model.resample(reso=[512] * 3, sigma_thresh=r.cfg.density_thresh, weight_thresh=r.cfg.weight_thresh / 512, dilate=2,
                     cameras=r._resample_cameras(), max_elements=r.cfg.max_grid_elements)
    t1.record()
    torch.cuda.synchronize()
    res["resample_ms"] = round(t0.elapsed_time(t1), 2)
    r.optimizer = type(r.optimizer)(r.model.density_data, r.model.sh_data, 0, 0, 0.95, 0.95)
    r.cfg.lambda_tv = r.cfg.lambda_tv_sh = 0.0
    res["reso_512"] = measure(r, a.steps, a.warmup, a.steps + a.warmup, ref)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
