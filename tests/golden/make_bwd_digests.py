#!/usr/bin/env python
"""Generates tests/golden/bwd_digests.json: SHA-256 digests of what one fused backward (ngp_network_bwd) writes -- the fp16 hash-grid
gradient and the fp32 weight gradients -- on seeded inputs at the lego (aabb 1) and fox (aabb 4) level tables, 2^19 entries per level.
The fused backward is deterministic, so any build must reproduce these bit for bit.  Needs an H100:

    python tests/golden/make_bwd_digests.py            # writes tests/golden/bwd_digests.json

Rows are ray-ordered like a training batch (runs of 64 samples along short random segments), so that cells repeat over consecutive
rows, and blocks of rows have a zero output gradient, so that the scatter skips rows.  The cases also cover a row count that is not a
multiple of the 256-row pair and a device-side live count below the launch size."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "bwd_digests.json")

# name -> (aabb_scale, rows launched, live rows read from the device or None, seed)
CASES = {
    "lego_2e18": (1, 1 << 18, None, 11),
    "lego_odd": (1, 100_003, None, 12),
    "fox_ndev": (4, 1 << 18, 200_001, 13),
}


def _mlp_weights(nhm, rng):
    shapes = [(64, 32)] + [(64, 64)] * nhm + [(16, 64)]
    lim = lambda s: np.sqrt(6.0 / (s[0] + s[1]))
    return np.concatenate([rng.uniform(-lim(s), lim(s), s).astype(np.float16).ravel() for s in shapes])


def inputs(n, n_params, seed):
    rng = np.random.default_rng(seed)
    n_seg = (n + 63) // 64
    a = rng.random((n_seg, 1, 3), dtype=np.float32)
    b = rng.random((n_seg, 1, 3), dtype=np.float32)
    t = np.linspace(0, 1, 64, dtype=np.float32).reshape(1, 64, 1)
    coords = np.zeros((n, 7), np.float32)
    coords[:, :3] = np.clip(a + (b - a) * t * np.float32(0.2), 0, 1).reshape(-1, 3)[:n]
    coords[:, 4:] = rng.random((n, 3), dtype=np.float32)
    grid = rng.uniform(-1, 1, n_params).astype(np.float16)
    wd, wr = _mlp_weights(0, rng), _mlp_weights(1, rng)
    dout = (rng.standard_normal((n, 4)) * 0.05).astype(np.float16)
    dout[(np.arange(n) // 5) % 9 == 0] = 0                              # runs of 5 rows without a gradient
    dout[rng.random(n) < 0.05] = 0                                      # and single ones
    return coords, grid, wd, wr, dout


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


_LEVELS = {}


def run_case(name):
    """Digests of grid_grad, dwd and dwr after one ngp_network_bwd from zeroed outputs.  The level tables stay alive: the backward
    sizes its fixed-point scratch when it first sees a table's device address, so a larger table allocated where a freed smaller one
    was would send its upper entries through the order-dependent fp16 path.  Run the cases in a process of their own for the same
    reason."""
    import torch
    from jnerf_b200 import ops
    aabb, n, n_live, seed = CASES[name]
    if aabb not in _LEVELS:
        _LEVELS[aabb] = ops.HashLevels(aabb, log2_hashmap_size=19)
    lv = _LEVELS[aabb]
    n_params = int(lv.offsets[-1]) * 2
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    coords, grid, wd, wr, dout = (cu(x) for x in inputs(n, n_params, seed))
    n_dev = None if n_live is None else torch.tensor([n_live], dtype=torch.int32, device="cuda")
    _, enc = ops.network_fwd(coords, grid, lv, wd, wr, n_dev=n_dev)
    gg = torch.zeros(n_params, dtype=torch.float16, device="cuda")
    dwd, dwr = torch.zeros(3072, device="cuda"), torch.zeros(7168, device="cuda")
    ops.network_bwd(coords, enc, lv, wd, wr, dout, gg, dwd, dwr, n_dev=n_dev)
    torch.cuda.synchronize()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    return {"grid_grad": digest(gg), "dwd": digest(dwd), "dwr": digest(dwr)}


def main(out):
    import torch
    sys.path.insert(0, os.path.join(HERE, "..", ".."))
    d = {"device": torch.cuda.get_device_name(0), "cases": {name: run_case(name) for name in CASES}}
    with open(out, "w") as f:
        json.dump(d, f, indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
