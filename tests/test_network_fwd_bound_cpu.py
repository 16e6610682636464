"""Rehearsal of the fused NGP forward's fp64 checks (ngp_fwd_ref, test_gpu_network_fwd_reference.py) on the CPU, against the oracle's
serial fp32 chain (orc_network_fwd with fp32 accumulation; hidden layers from orc_mlp_fwd).  The oracle is another fp32 evaluation of
the same network, in another summation order, so each of its outputs and hidden activations must lie in the interval, and it must agree
with the mirror on every tile as often as the GPU test requires of the kernel.  The checks must also fail for the faults they are there
to catch: a hidden layer that rounds toward zero, a tile's rows permuted, and the blue channel taken from green."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle_lib as ol
from ngp_fwd_ref import (interval_chain, interval_check, probe_expected, probe_sets, probe_weights, rn16, sh_f32, sh_f64, sh_interval,
                         split_weights, tile_agreement)
from test_gpu_network_fwd_reference import DENSITY_FLOOR, RGB_FLOOR

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_bwd_digests import inputs as ray_inputs  # noqa: E402

N = 4096 + 77


def _regime(name, seed=5):
    cfg = ol.HashCfg(1, log2_hashmap_size=19)
    coords, grid, wd, wr, _ = ray_inputs(N, cfg.n_params, seed)
    if name == "tiny":
        grid = (grid.astype(np.float32) * np.float32(1e-5)).astype(np.float16)
    elif name == "big":
        wd, wr = wd * np.float16(2), wr * np.float16(2)
    return cfg, coords, grid, wd, wr


def _oracle(cfg, coords, grid, wd, wr):
    """(out, enc, sh16, hidden) of the oracle's serial fp32 chain"""
    pos, dirs = coords[:, :3].copy(), coords[:, 4:].copy()
    out, enc, h = ol.network_fwd(cfg, pos, dirs, grid, wd, wr, acc32=True)
    sh16 = ol.sh(dirs, np.float16)
    h2_, inter_d = ol.mlp_fwd(wd, enc, 0)
    assert np.array_equal(h2_.view(np.uint16), h.view(np.uint16))
    _, inter_r = ol.mlp_fwd(wr, np.concatenate([h, sh16], 1), 1)
    n = coords.shape[0]
    hidden = dict(hd=inter_d, h=h, h1=inter_r[:n], h2=inter_r[n:])
    return out, enc, sh16, hidden


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def _chain(enc, sh16, dirs, wd, wr):
    lo, hi = sh_interval(dirs)
    return interval_chain(_t(enc), _t(sh16), lo, hi, _t(wd), _t(wr))


@pytest.mark.parametrize("regime", ["ref", "tiny", "big"])
def test_oracle_lies_in_the_intervals_and_meets_the_floors(regime):
    cfg, coords, grid, wd, wr = _regime(regime)
    out, enc, sh16, hidden = _oracle(cfg, coords, grid, wd, wr)
    ch = _chain(enc, sh16, coords[:, 4:], wd, wr)
    inside, ratio = interval_check(_t(out), ch)
    assert bool(inside.all()), f"{int((~inside).sum())} oracle outputs outside their interval, worst ratio {float(ratio.max()):.3g}"
    for name, (x, lo, hi) in ch["hidden"].items():
        g = _t(hidden[name]).to(torch.float64)
        assert bool(((g >= lo) & (g <= hi)).all()), f"oracle {name} outside its interval"
    share = tile_agreement(_t(out), ch["out"]).min(0).values
    print(f"[fwd-cpu] {regime}: worst ratio {[round(float(v), 3) for v in ratio.max(0).values]}, radius median/max "
          f"{float((ch['hi'] - ch['lo'])[:, :3].median()) / 2:.3g}/{float(torch.maximum(ch['hi'] - ch['out'], ch['out'] - ch['lo']).max()):.3g}, "
          f"lowest tile agreement {[round(float(v), 4) for v in share]}")
    assert float(share[:3].min()) >= RGB_FLOOR and float(share[3]) >= DENSITY_FLOOR, share


def _rz16(y):
    """float64 -> the float64 value of the fp16 next to y toward zero (__float2half_rz), finite range"""
    a = y.abs()
    q = torch.exp2((torch.frexp(a).exponent.to(torch.float64) - 11).clamp_min(-24))
    return torch.copysign(torch.floor(a / q) * q, y)


def test_a_layer_rounding_toward_zero_fails_the_floor():
    """The mirror with one hidden layer rounded toward zero instead of to nearest: within the interval, below the agreement floor."""
    cfg, coords, grid, wd, wr = _regime("ref")
    out, enc, sh16, _ = _oracle(cfg, coords, grid, wd, wr)
    ch = _chain(enc, sh16, coords[:, 4:], wd, wr)
    W0d, Woutd, W0r, W1r, Woutr = split_weights(_t(wd), _t(wr))
    hd = rn16(torch.relu(_t(enc).double() @ W0d.T))
    h = rn16(hd @ Woutd.T)
    for bad in ("h1", "h2"):
        h1 = torch.relu(torch.cat([h, _t(sh16).double()], 1) @ W0r.T)
        h1 = _rz16(h1) if bad == "h1" else rn16(h1)
        h2 = torch.relu(h1 @ W1r.T)
        h2 = _rz16(h2) if bad == "h2" else rn16(h2)
        faulty = torch.cat([rn16(h2 @ Woutr[:3].T), h[:, :1]], 1)
        share = tile_agreement(faulty, ch["out"]).min(0).values
        assert float(share[:3].max()) < RGB_FLOOR, (bad, share)
        assert float(share[3]) == 1.0                                     # the density output does not pass through the colour net


def test_permuted_tile_and_wrong_channel_fail_the_interval():
    cfg, coords, grid, wd, wr = _regime("ref")
    out, enc, sh16, _ = _oracle(cfg, coords, grid, wd, wr)
    ch = _chain(enc, sh16, coords[:, 4:], wd, wr)
    o = _t(out)
    perm = o.clone()
    perm[3 * 128:4 * 128] = o[3 * 128:4 * 128].roll(1, 0)               # one tile's rows rotated by one
    inside, _ = interval_check(perm, ch)
    assert int((~inside[3 * 128:4 * 128]).any(1).sum()) > 64
    blue = o.clone()
    blue[:, 2] = o[:, 1]
    inside, _ = interval_check(blue, ch)
    assert float((~inside[:, 2]).double().mean()) > 0.5


@pytest.mark.parametrize("regime", ["ref", "tiny"])
def test_probe_weights_route_exactly_on_the_oracle(regime):
    cfg, coords, grid, _, _ = _regime(regime)
    pos, dirs = coords[:, :3].copy(), coords[:, 4:].copy()
    sh16 = ol.sh(dirs, np.float16)
    reached = set()
    for k0, srcs in probe_sets():
        wd, wr = probe_weights(k0, srcs)
        out, enc, _ = ol.network_fwd(cfg, pos, dirs, grid, wd, wr, acc32=True)
        want = probe_expected(k0, srcs, _t(enc), _t(sh16))
        assert torch.equal(_t(out).double(), want.double()), (k0, srcs)
        reached |= {("enc", k0)} | {("enc", k) if k is not None else ("sh", c - 16) for c, k in srcs} | {("h", c) for c, k in srcs if c < 16}
    assert reached >= {("enc", k) for k in range(32)} | {("sh", k) for k in range(16)} | {("h", c) for c in range(1, 16)}


def test_sh_bound_holds_for_fp32_evaluations():
    """The oracle's fp32 SH, and the contracted evaluation of the fused kernels, lie within the fp32 evaluation bound of the float64 basis,
    on random directions and on directions built from the components 0, 0.25, 0.5, 1 and their neighbours (where x, y, z are 0 or +-1
    and the cancelling terms vanish exactly)."""
    rng = np.random.default_rng(11)
    special = np.float32([0, 0.25, 0.5, 1])
    special = np.concatenate([special, np.nextafter(special, np.float32(2)), np.nextafter(special, np.float32(-1))[1:]])
    grid3 = np.stack(np.meshgrid(special, special, special, indexing="ij"), -1).reshape(-1, 3)
    dirs = np.concatenate([grid3, rng.random((50_000, 3), dtype=np.float32), rng.choice(special, (5000, 3))]).astype(np.float32)
    v, e = sh_f64(dirs)
    o32 = ol.sh(dirs, np.float32)
    assert np.array_equal(sh_f32(dirs, contract=False).view(np.uint32), o32.view(np.uint32))     # the emulation is the oracle's C
    for name, got in (("oracle", o32), ("contracted", sh_f32(dirs))):
        err = (torch.from_numpy(got.astype(np.float64)) - v).abs()
        assert bool((err <= e).all()), f"{name}: {int((err > e).sum())} SH values outside the bound, worst {float((err / e).max()):.3g}"
    lo, hi = sh_interval(dirs)
    for got in (ol.sh(dirs, np.float16), sh_f32(dirs).astype(np.float16)):
        g = torch.from_numpy(got.astype(np.float64))
        assert bool(((g >= lo) & (g <= hi)).all())
