"""Per-kernel timings (CUDA events, L2 flushed between iterations) for the hot-path operators at BASELINE sizes.
Usage: python tools/microbench.py [N]   -- prints one line per kernel with algorithmic GB/s or TFLOP/s."""
import sys
import os
import json
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jnerf_b200 import ops  # noqa: E402

PEAKS = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}                         # H100 SXM data sheet; MEASURED_PEAKS.json overrides
try:
    PEAKS.update(json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))))
except Exception:
    pass


def timeit(fn, iters=20, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.sum()            # read-only sweep > L2: evicts without leaving dirty lines to write back
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2] * 1e-3


def main():
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 262144
    dev = "cuda"
    torch.manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # > 50 MB L2
    lv = ops.HashLevels(1)
    grid = (torch.rand(lv.n_params, device=dev) * 2e-4 - 1e-4).half()
    x = torch.rand(N, 3, device=dev)
    coords = torch.zeros(N, 7, device=dev)
    coords[:, :3] = x
    coords[:, 4:] = torch.rand(N, 3, device=dev)
    wd = (torch.rand(3072, device=dev) - 0.5).half()
    wr = (torch.rand(7168, device=dev) - 0.5).half()
    res = {}

    def rep(name, t, bytes_=None, flops=None):
        s = f"{name:28s} {t*1e6:9.1f} us"
        if bytes_:
            s += f"  {bytes_/t/1e9:9.1f} GB/s algorithmic ({bytes_/t/1e9/PEAKS['hbm_gbs']*100:5.1f}% of measured HBM)"
        if flops:
            s += f"  {flops/t/1e12:8.2f} TFLOP/s ({flops/t/1e12/PEAKS['bf16_tflops']*100:5.2f}% of measured bf16)"
        print(s, flush=True)
        res[name] = t

    for nm, fl in (("hot-L2", None), ("flushed", flush)):
        rep(f"hash_fwd f16 [{nm}]", timeit(lambda: ops.hash_fwd(x, grid, lv), flush=fl), bytes_=N * 588)
    dy = (torch.randn(N, 32, device=dev) * 1e-3).half()
    gg = torch.empty(lv.n_params, dtype=torch.float16, device=dev)
    rep("hash_bwd f16 (+memset)", timeit(lambda: ops.hash_bwd(x, dy, lv, gg), flush=flush), bytes_=N * 1100 + lv.n_params * 2)
    X = torch.randn(N, 32, device=dev).half()
    rep("mlp_fwd 32-64-64-16", timeit(lambda: ops.mlp_fwd(wr, X, 1), flush=flush), flops=N * 2 * (32 * 64 + 64 * 64 + 64 * 16))
    Y, inter = ops.mlp_fwd(wr, X, 1)
    dY = torch.randn(N, 16, device=dev).half()
    rep("mlp_bwd 32-64-64-16", timeit(lambda: ops.mlp_bwd(wr, X, inter, dY, 1, 3), flush=flush), flops=N * 4 * (32 * 64 + 64 * 64 + 64 * 16))
    out = torch.empty(N, 4, dtype=torch.float16, device=dev)
    enc = torch.empty(N, 32, dtype=torch.float16, device=dev)
    rep("network_fwd fused", timeit(lambda: ops.network_fwd(coords, grid, lv, wd, wr, out=out, enc=enc), flush=flush), bytes_=N * (524 + 28 + 8 + 64),
        flops=N * 20480)
    dout = (torch.randn(N, 4, device=dev) * 1e-3).half()
    dwd = torch.zeros(3072, device=dev)
    dwr = torch.zeros(7168, device=dev)
    rep("network_bwd fused", timeit(lambda: ops.network_bwd(coords, enc, lv, wd, wr, dout, gg, dwd, dwr), flush=flush),
        bytes_=N * (64 + 28 + 8 + 128 * 8), flops=N * 61440)
    m = torch.zeros(lv.n_params, device=dev)
    v = torch.zeros(lv.n_params, device=dev)
    ms = grid.float()
    rep("adam_ema 12.2M f16", timeit(lambda: ops.adam_ema(grid, gg, m, v, ms, 0.1, 5), flush=flush), bytes_=lv.n_params * 30)
    pos = x.contiguous()
    rep("density_fwd", timeit(lambda: ops.density_fwd(pos, grid, lv, wd), flush=flush), bytes_=N * (524 + 12 + 2))
    print("timeout flag:", ops.lib.load().ngp_debug_timeout_flag())


if __name__ == "__main__":
    main()
