"""The reference defines its MLP twice: the prebuilt tiny-cuda-nn object (fp16 accumulators: every tensor instruction in
fully_fused_mlp_function.o is HMMA.*.F16) and the nn.Linear fallback
(models/networks/ngp_network.py:59-67, wide accumulation).  The oracle and the CUDA kernels follow the second.  This test restates
the first as a numerical MODEL (fp16 rounding of the accumulator after every 16-wide K block) and measures how far apart the two
definitions are on NGP-shaped inputs: that distance is the floor under any float tolerance for R7, and the tolerance the GPU
parity tests use (6e-3 absolute on O(1) outputs, tests/test_gpu_ops.py) sits above it."""
import numpy as np

import oracle_lib as ol


def mlp_f16_accumulate(W, X, nhm, kblock=16):
    """Forward pass with the accumulator held in fp16 between K blocks (HMMA.16816.F16 D=A*B+C with C, D in fp16)."""
    shapes = [(64, 32)] + [(64, 64)] * nhm + [(16, 64)]
    h, o = X.astype(np.float16), 0
    for li, (out_f, in_f) in enumerate(shapes):
        w = W[o:o + out_f * in_f].reshape(out_f, in_f).astype(np.float32)
        o += out_f * in_f
        acc = np.zeros((h.shape[0], out_f), np.float16)
        for k in range(0, in_f, kblock):
            acc = (acc.astype(np.float32) + h[:, k:k + kblock].astype(np.float32) @ w[:, k:k + kblock].T).astype(np.float16)
        h = np.maximum(acc, np.float16(0)) if li < len(shapes) - 1 else acc
    return h


def test_distance_between_the_references_two_mlp_definitions():
    rng = np.random.default_rng(0)
    for nhm in (0, 1):
        shapes = [(64, 32)] + [(64, 64)] * nhm + [(16, 64)]
        W = np.concatenate([rng.uniform(-np.sqrt(6 / sum(s)), np.sqrt(6 / sum(s)), s).astype(np.float16).ravel() for s in shapes])
        X = np.clip(rng.standard_normal((4096, 32)), -4, 4).astype(np.float16)
        wide, _ = ol.mlp_fwd(W, X, nhm)                          # the oracle: nn.Linear semantics
        narrow = mlp_f16_accumulate(W, X, nhm)
        d = np.abs(wide.astype(np.float32) - narrow.astype(np.float32))
        scale = np.abs(wide.astype(np.float32)).max()
        assert scale > 0.5
        # the two reference definitions agree to a few fp16 ulps of the output range and not better
        assert d.max() <= 6e-3 * max(1.0, scale), (d.max(), scale)
        assert d.max() > 0, "an fp16 accumulator must differ somewhere"
        assert d.mean() <= 1e-3
