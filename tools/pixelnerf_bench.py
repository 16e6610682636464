"""Times one pixelNeRF training step at 2048 rays x 64 samples x 3 reference views: the fused path (csrc/pixelnerf.cu) against the same
network as fp16 nn.Linear + autograd (cuBLAS) + torch grid_sample, both around the same composite kernel and Adam.  Prints one JSON line
with per-stage CUDA-event times, achieved TFLOP/s from the shape formulas, and the GPU's name, power limit and SM clock.
--train N: also trains N steps on a capture and reports the held-out PSNR for pixel_aligned False and True, and the test / video wall time.

    python tools/pixelnerf_bench.py [--data tests/golden/pixelnerf_tiny.npz] [--iters 20] [--train 0]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jnerf_b200 import ops  # noqa: E402
from jnerf_b200.plugin import pixelnerf as pn  # noqa: E402

R, S, NREF, W = 2048, 64, 3, 512


def flops():
    """(forward, backward) multiply-add FLOPs of one step from the shapes: per sample the stem (42 x 512) and the head (512 x 4) once,
    per reference row the three f1 blocks of three 512 x 512 layers, per sample the two f2 blocks of two; the backward is dgrad + wgrad of
    every layer except the first layer's dgrad."""
    Ms, M3 = R * S, R * S * NREF
    f = 2 * (Ms * 42 * W + M3 * 9 * W * W + Ms * 4 * W * W + Ms * W * 4)
    b = 2 * (Ms * 42 * W + 2 * M3 * 9 * W * W - M3 * 3 * W * W + 2 * Ms * 4 * W * W + 2 * Ms * W * 4)
    return f, b


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "pixelnerf_tiny.npz"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--train", type=int, default=0)
    a = ap.parse_args()
    data = pn.TinyNerfData(a.data, 3)
    ref = pn.ReferenceViews(data.images[:3], data.poses[:3], data.focal, pn.ImageEncoder(seed=0))
    g = torch.Generator(device="cuda").manual_seed(0)
    batch = next(iter(data.batches(R, g)))
    rays, target = batch[:, :6].contiguous(), batch[:, 6:9].contiguous()
    z = 2.0 + 4.0 * (torch.linspace(0, 1, S + 1, device="cuda")[:-1] + 0.5 / S)
    m = pn.PixelNeRF(seed=0)
    saved = torch.empty(ops.pixelnerf_workspace_bytes(R * S, NREF)[0], dtype=torch.uint8, device="cuda")
    st = {}

    def fused_fwd():
        st["raw"] = ops.pixelnerf_fwd(rays, z, m.params, ref.feats, ref.cams, ref.scale, saved=saved)

    def fused_loss():
        st["draw"] = ops.pixelnerf_composite_loss_bwd(st["raw"], z, rays, target, grad_scale=float(R))[2]

    def fused_bwd():
        st["grad"] = ops.pixelnerf_bwd(R, S, m.params, ref.feats, saved, st["raw"], st["draw"])

    def adam():
        ops.adam_ema(m.params, st["grad"], m.m, m.v, m.master, 0.0, 1, 0.9, 0.999, 1e-8, 0.0, grad_scale=1.0 / R, zero_grad=False)

    def fused_step():
        fused_fwd(); fused_loss(); fused_bwd(); adam()

    # the cuBLAS chain: fp16 nn.Linear weights, autograd, torch grid_sample on the channel-first maps
    state = {k: v.cuda().half().requires_grad_() for k, v in m.reference_state().items()}
    feats_cf = ref.feats.permute(0, 3, 1, 2).contiguous()
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[None, :, None]).reshape(-1, 3)
    dirs = rays[:, None, 3:6].expand(-1, S, -1).reshape(-1, 3)

    def torch_step():
        enc = pn.positional_encoding(pts, dirs).half()
        uv = pn.project(pts, ref.cams, ref.scale).half()
        feat = torch.nn.functional.grid_sample(feats_cf, uv[:, :, None, :], align_corners=True, padding_mode="border")[..., 0].permute(0, 2, 1)
        raw = pn.network_torch(state, enc, feat, torch.float16)
        draw = ops.pixelnerf_composite_loss_bwd(raw.detach().contiguous(), z, rays, target, grad_scale=float(R))[2]
        for v in state.values():
            v.grad = None
        raw.backward(draw)
        grad = pn.pack({k: v.grad for k, v in state.items()})
        ops.adam_ema(m.params, grad, m.m, m.v, m.master, 0.0, 1, 0.9, 0.999, 1e-8, 0.0, grad_scale=1.0 / R, zero_grad=False)

    fused_step()
    ms = {"fwd": timed(fused_fwd, a.iters), "loss": timed(fused_loss, a.iters), "bwd": timed(fused_bwd, a.iters), "adam": timed(adam, a.iters)}
    ms["step"] = timed(fused_step, a.iters)
    ms["torch_step"] = timed(torch_step, a.iters)
    ms["step_again"] = timed(fused_step, a.iters)
    ff, fb = flops()
    out = {"metric": "pixelnerf_train_step", "rays": R, "samples": S, "n_ref": NREF, "ms": {k: round(v, 3) for k, v in ms.items()},
           "tflops_fwd": round(ff / ms["fwd"] / 1e9, 1), "tflops_bwd": round(fb / ms["bwd"] / 1e9, 1),
           "tflops_step": round((ff + fb) / ms["step"] / 1e9, 1), "speedup_vs_torch": round(ms["torch_step"] / ms["step"], 2),
           "gpu": gpu_info(), "max_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    if a.train:
        from jnerf_b200.pixelnerf_runner import PixelNeRFRunner, pixelnerf_cfg
        from jnerf_b200.utils.config import get_cfg, update_cfg
        for pa in (False, True):
            get_cfg().clear()
            update_cfg(**pixelnerf_cfg(a.data, pixel_aligned=pa, log_dir=tempfile.mkdtemp()))
            r = PixelNeRFRunner()
            p0 = r.test()
            t0 = time.time()
            r.train(steps=a.train)
            torch.cuda.synchronize()
            t_train = time.time() - t0
            t0 = time.time()
            p1 = r.test()
            t_test = time.time() - t0
            t0 = time.time()
            r.render()
            t_video = time.time() - t0
            out[f"psnr_pixel_aligned_{pa}"] = {"encoder": r.encoder_label, "steps": a.train, "before": round(p0, 3), "after": round(p1, 3),
                                               "train_s": round(t_train, 2), "test_s": round(t_test, 2), "video_s": round(t_video, 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
