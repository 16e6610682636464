#!/usr/bin/env python
"""SURVEY.md 8d(ii): the reference's own kernels, compiled UNMODIFIED for sm_90a with the reference's launch shapes
(oracle/_ref/libref_gpu_constdt.so, recipe oracle/Makefile), timed and compared against this library on the same H100 and the
same inputs -- "the kernel to beat" for R2, R3, R6, R8, R9.

    python tools/ref_gpu_compare.py [--steps 300] [--out gpurun_out/ref_gpu_compare.json]

Inputs come from a short real training run (trained occupancy grid, a ray batch, ray-ordered samples, real network outputs).
Timing: CUDA events, median of 15 launches after 3 warm-ups.  Benchmark infrastructure, not product code."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref", "libref_gpu_constdt.so")

VP, U32, U64, F32, I32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float, C.c_int
SIG = {
    "refgpu_hash_fwd_f16_constdt": [U32, VP, VP, VP, F32, VP, VP, VP],
    "refgpu_hash_bwd_f16_constdt": [U32, VP, VP, VP, F32, VP, VP, U64],
    "refgpu_march_constdt": [U32, F32, F32, U32, VP, VP, VP, F32, VP, VP, VP, VP, VP, VP, VP, F32, U64, U64, I32],
    "refgpu_rgb_fwd_f16_constdt": [U32, VP, VP, VP, VP, VP, VP],
    "refgpu_rgb_bwd_f16_constdt": [U32, U32, VP, VP, VP, VP, VP, VP, VP],
}


def load_ref():
    lib = C.CDLL(REF)
    for name, args in SIG.items():
        f = getattr(lib, name)
        f.argtypes, f.restype = args, C.c_int
    return lib


def p(t):
    return t.data_ptr()


def timeit(fn, iters=15, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "ref_gpu_compare.json"))
    args = ap.parse_args()
    from jnerf_b200 import lib as nlib, ops, plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    nlib.load()
    ref = load_ref()
    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=1))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 20
    cfg.dataset.train.H = cfg.dataset.train.W = 400
    cfg.dataset.val = None
    cfg.dataset.train.pop("root_dir", None)
    r = Runner()
    for _ in range(args.steps):
        r.train_step()
    torch.cuda.synchronize()
    s, m, ds = r.sampler, r.model, r.dataset["train"]
    res = {"config": f"lego stand-in after {args.steps} steps; reference kernels = oracle/_ref/libref_gpu_constdt.so (unmodified sources, sm_90a, reference launch shapes)",
           "unit": "us (median of 15)"}

    def section(name, fn):
        try:
            res[name] = fn()
        except Exception as e:                       # keep the other sections
            res[name] = {"error": repr(e)[:300]}
        print(name, json.dumps(res[name]), flush=True)

    # ------------------------------------------------------------------ a ray batch
    R = int(s.n_rays_per_batch)
    pix = ds.next_pixels(R)
    img_ids, rays_o, rays_d = ds.rays_for(pix)
    rays_o, rays_d = rays_o.contiguous(), rays_d.contiguous()
    rng = s.rng.copy()
    max_samples = R * 1024
    coords_o = torch.empty((max_samples, 7), device="cuda")
    ws = torch.empty(int(nlib.load().ngp_march_workspace_bytes(R)), dtype=torch.uint8, device="cuda")

    def our_march():
        return ops.march(rays_o, rays_d, s.density_grid_bitfield, s.aabb_range, max_samples, s.cone_angle_constant, s.near_distance,
                         s.NERF_CASCADES, s.const_dt, rng, coords=coords_o, workspace=ws)

    coords_r = torch.zeros((max_samples, 7), device="cuda")
    cnt_r = torch.zeros(2, dtype=torch.int32, device="cuda")
    idx_r = torch.zeros(R, dtype=torch.int32, device="cuda")
    ns_r = torch.zeros((R, 2), dtype=torch.int32, device="cuda")

    def ref_march(memset=1):
        rc = ref.refgpu_march_constdt(R, s.aabb_range[0], s.aabb_range[1], max_samples, p(rays_o), p(rays_d), p(s.density_grid_bitfield),
                                      s.cone_angle_constant, p(ds.metadata), p(img_ids), p(cnt_r), p(idx_r), p(ns_r), p(coords_r),
                                      p(ds.transforms_gpu), s.near_distance, int(rng[0]), int(rng[1]), memset)
        assert rc == 0, rc

    def march_section():
        _, _, ns_o, cnt_o = our_march()
        ref_march()
        torch.cuda.synchronize()
        n_o, n_r = ns_o[:, 0].long(), ns_r[:, 0].long()
        same_counts = bool(torch.equal(n_o, n_r))
        total = int(n_o.sum())
        ray_of = torch.repeat_interleave(torch.arange(R, device="cuda"), n_o)
        k = torch.arange(total, device="cuda") - torch.repeat_interleave(ns_o[:, 1].long(), n_o)
        rows_o = coords_o[ns_o[ray_of, 1].long() + k]
        rows_r = coords_r[ns_r[ray_of, 1].long() + k] if same_counts else None
        bit_equal = bool(same_counts and torch.equal(rows_o.view(torch.int32), rows_r.view(torch.int32)))
        return {"rays": R, "samples": total, "per_ray_counts_identical": same_counts, "every_sample_bit_identical": bit_equal,
                "ours_us": timeit(our_march), "reference_us": timeit(lambda: ref_march(1)),
                "reference_without_its_117MB_memset_us": timeit(lambda: ref_march(0))}

    section("march (R6)", march_section)

    # ------------------------------------------------------------------ ray-ordered samples of this batch (our compaction)
    _, _, ns_o, _ = our_march()
    cap = s.target_batch_size
    _, ns_c, cnt_c = ops.compact(coords_o, ns_o, cap, alias=True)
    N = min(int(cnt_c[0]), cap)
    coords = coords_o[:cap]
    pos = coords[:N, :3].contiguous()
    lv = m.pos_encoder.levels
    grid = m.pos_encoder.m_grid.data
    offsets_dev = torch.from_numpy(lv.offsets.astype(np.uint32).view(np.int32).copy()).cuda()
    pos_soa = torch.empty(3 * N, device="cuda")
    enc_soa = torch.empty((16 * N, 2), dtype=torch.float16, device="cuda")
    out_r = torch.empty((N, 32), dtype=torch.float16, device="cuda")

    def ref_hash_fwd():
        rc = ref.refgpu_hash_fwd_f16_constdt(N, p(pos), p(grid), p(offsets_dev), lv.log2_per_level_scale, p(pos_soa), p(enc_soa), p(out_r))
        assert rc == 0, rc

    def hash_fwd_section():
        ref_hash_fwd()
        out_o = ops.hash_fwd(pos, grid, lv)
        torch.cuda.synchronize()
        d = (out_o.float() - out_r.float()).abs()
        sc = out_r.float().abs().max().item()
        return {"points": N, "max_abs_diff_over_max": d.max().item() / sc, "mean_abs_diff_over_max": d.mean().item() / sc,
                "ours_standalone_us": timeit(lambda: ops.hash_fwd(pos, grid, lv)), "reference_us": timeit(ref_hash_fwd)}

    section("hash forward (R2), ray-ordered samples", hash_fwd_section)

    dy = (torch.randn((N, 32), device="cuda") * 1e-3).half()
    dy_soa = torch.empty((16 * N, 2), dtype=torch.float16, device="cuda")
    gg_r = torch.empty(grid.numel(), dtype=torch.float16, device="cuda")
    gg_o = torch.zeros(grid.numel(), dtype=torch.float16, device="cuda")

    def ref_hash_bwd():
        rc = ref.refgpu_hash_bwd_f16_constdt(N, p(pos_soa), p(dy), p(offsets_dev), lv.log2_per_level_scale, p(dy_soa), p(gg_r), grid.numel())
        assert rc == 0, rc

    def our_hash_bwd():
        gg_o.zero_()
        ops.hash_bwd(pos, dy, lv, grid_grad=gg_o)

    def hash_bwd_section():
        ref_hash_fwd()                                # fills pos_soa as the reference's forward does
        ref_hash_bwd()
        our_hash_bwd()
        torch.cuda.synchronize()
        d = (gg_o.float() - gg_r.float()).abs()
        sc = gg_r.float().abs().max().item()
        return {"points": N, "max_abs_diff_over_max": d.max().item() / sc, "mean_abs_diff_over_max": d.mean().item() / sc,
                "note": "the reference accumulates with fp16 atomics (order-dependent rounding); ours combines runs in fp32 first",
                "ours_standalone_incl_zeroing_us": timeit(our_hash_bwd), "reference_incl_memset_us": timeit(ref_hash_bwd)}

    section("hash backward (R3), ray-ordered samples", hash_bwd_section)

    # ------------------------------------------------------------------ fused network (what a training step launches)
    wd, wr = m.density_mlp.con_weights.data, m.rgb_mlp.con_weights.data
    net, enc = ops.network_fwd(coords, grid, lv, wd, wr, n_dev=cnt_c[0:1])

    def fused_section():
        dnet = (torch.randn((cap, 4), device="cuda") * 1e-3).half()
        gg = torch.zeros(grid.numel(), dtype=torch.float16, device="cuda")
        dwd, dwr = torch.zeros(wd.numel(), device="cuda"), torch.zeros(wr.numel(), device="cuda")
        return {"samples": N,
                "ours_fused_hash+SH+both_MLPs_forward_us": timeit(lambda: ops.network_fwd(coords, grid, lv, wd, wr, n_dev=cnt_c[0:1], out=net, enc=enc)),
                "ours_fused_MLP_backward+hash_scatter_us": timeit(lambda: ops.network_bwd(coords, enc, lv, wd, wr, dnet, gg, dwd, dwr, n_dev=cnt_c[0:1])),
                "note": "the reference's MLP exists only as sm_75/80/86 SASS and cannot run on sm_90; compare against its hash kernels alone above"}

    section("fused network (R2+R4+R7 / R7+R3)", fused_section)

    # ------------------------------------------------------------------ composite
    bg = torch.rand((R, 3), device="cuda")
    rgb_r = torch.empty((R, 3), device="cuda")
    loss_grad = (torch.randn((R, 3), device="cuda") * 1e-2)
    mean = s.density_grid_mean
    dnet_r = torch.empty((cap, 4), dtype=torch.float16, device="cuda")

    def ref_rgb_fwd():
        rc = ref.refgpu_rgb_fwd_f16_constdt(R, p(net), p(coords), p(ns_o), p(rgb_r), p(ns_c), p(bg))
        assert rc == 0, rc

    def ref_rgb_bwd():
        rc = ref.refgpu_rgb_bwd_f16_constdt(R, cap, p(dnet_r), p(net), p(ns_c), p(coords), p(loss_grad), p(rgb_r), p(mean))
        assert rc == 0, rc

    def composite_section():
        ref_rgb_fwd()
        rgb_o = ops.composite_fwd(net, coords, ns_o, ns_c, bg)
        ref_rgb_bwd()
        dnet_o = ops.composite_bwd(net, coords, ns_c, loss_grad, rgb_r, mean)
        torch.cuda.synchronize()
        target = torch.rand((R, 3), device="cuda")
        dd = (dnet_o[:N].float() - dnet_r[:N].float()).abs()
        return {"rays": R, "samples": N, "rgb_max_abs_diff": (rgb_o - rgb_r).abs().max().item(),
                "dnet_max_abs_diff_over_max": dd.max().item() / max(dnet_r[:N].float().abs().max().item(), 1e-30),
                "ours_forward_us": timeit(lambda: ops.composite_fwd(net, coords, ns_o, ns_c, bg)), "reference_forward_us": timeit(ref_rgb_fwd),
                "ours_backward_us": timeit(lambda: ops.composite_bwd(net, coords, ns_c, loss_grad, rgb_r, mean)),
                "reference_backward_incl_memset_us": timeit(ref_rgb_bwd),
                "ours_fused_forward+huber+backward_us": timeit(lambda: ops.composite_loss_bwd(net, coords, ns_o, ns_c, bg, target, mean))}

    section("composite (R8, R9)", composite_section)

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
