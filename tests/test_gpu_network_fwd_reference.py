"""The fused NGP forward (network_fwd_kernel: ngp_network_fwd, ngp_density_fwd, ngp_density_lattice) against float64 references at
training batch sizes, entry by entry (ngp_fwd_ref has the references and the derivations).

Per case, with realistic weights:
- the saved encoding equals the oracle's fp32-accumulated encoding (orc_hash_fwd_f16_acc32) bit for bit, on both of its store paths
  (TMA tensor stores when enc is 16-byte aligned, per-row stores from the gather warps otherwise);
- (a) every output entry lies in its rigorous interval, no outliers;
- (b) on every 128-row tile with at least 64 live rows, at least RGB_FLOOR of each colour column and DENSITY_FLOOR of the density
  column equal the float64 mirror bit for bit.  A whole wrong tile cannot hide in a batch average, and a hidden layer rounding toward
  zero drops the colour shares to 22-40 % (test_network_fwd_bound_cpu.py);
- ngp_density_fwd equals column 3 bit for bit, and repeated launches give identical bits.
And with fourteen routing-probe weight sets (ngp_fwd_ref.probe_sets) that make every product and sum exact, each output equals the
encoded feature, density-net output or SH feature routed to it, bit for bit on every row.  This is the check that pins tile, buffer,
lane and column routing exactly.

SH.  The mirror's SH centre is the fused kernels' own fp32 evaluation, with seven terms contracted to FMA as nvcc compiles them
(ngp_fwd_ref.sh_f32); the routed SH features must equal it bit for bit and lie in the float64 SH interval.  The oracle's unfused SH
(ol.sh) differs from the kernel's in the last fp16 bit on about one feature in 12 000; the count is printed per case.

Floors.  Measured on an H100 80GB HBM3 (700 W power limit) over the fourteen cases below, the lowest per-tile shares were 0.953 (colour)
and 0.977 (density), i.e. at most 6 and 3 flips in a 128-row tile.  The floors, 0.90 and 0.94, allow 12 and 7: at the flip rates seen
(about 0.5 % of colour and 0.15 % of density entries) a tile falls below them with a probability under 1e-8, while a wrong tile, lane,
column or rounding mode takes a column's share far below (test_network_fwd_bound_cpu.py: 22-40 % for a colour layer rounding toward
zero).  The worst interval ratios were 0.81 (colour, on the trained table) and 0.87 (density); the colour radii have a median of 5-64
fp16 ulps, the density radii one.

Live rows.  For rows at or past the live count n_dev: `out` rows are never written; `enc` rows past the last live tile are never
written; rows of the last live tile past n_dev may be written by the TMA path (its 128-row box is clipped only at n_max), never by the
per-row path."""
import os
import sys
import time

import numpy as np
import pytest
import torch

import oracle_lib as ol
from ngp_fwd_ref import (ROWS, interval_chain, interval_check, probe_expected, probe_sets, probe_weights, radius_ulps, sh_f32, sh_interval,
                         tile_agreement)
from test_gpu_ops import device_scales

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_bwd_digests import inputs as ray_inputs  # noqa: E402

pytestmark = pytest.mark.gpu

RGB_FLOOR, DENSITY_FLOOR = 0.90, 0.94
SENTINEL = 0x7E5A                     # an fp16 NaN payload the kernel never produces
N_MAX = 1 << 18

_TABLES = {}


def _levels(aabb):
    from jnerf_b200 import ops
    if aabb not in _TABLES:
        _TABLES[aabb] = (ops.HashLevels(aabb, log2_hashmap_size=19), ol.HashCfg(aabb, log2_hashmap_size=19))
    return _TABLES[aabb]


def _sm():
    from jnerf_b200 import ops
    return int(ops.lib.load().ngp_sm_count())


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _filled(shape, off=0):
    """an fp16 tensor of `shape` holding SENTINEL, starting `off` halfs into a larger buffer (off = 4: 8 bytes, not 16-byte aligned)"""
    n = int(np.prod(shape))
    buf = torch.full((n + 8,), SENTINEL, dtype=torch.int16, device="cuda").view(torch.float16)
    return buf[off:off + n].view(*shape)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _fwd(coords, grid, lv, wd, wr, n_dev=None, off=0):
    from jnerf_b200 import ops
    n = coords.shape[0]
    out, enc = _filled((n, 4)), _filled((n, 32), off)
    ops.network_fwd(coords, grid, lv, wd, wr, n_dev=n_dev, out=out, enc=enc)
    torch.cuda.synchronize()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    return out, enc


# ------------------------------------------------------------------------------------------------ cases
def _march_rows(seed=21):
    """a training batch from the march: 8192 rays through a spherical shell, compacted at the 2^18 cap; n_dev is the march's raw sample
    count, which exceeds the cap"""
    from jnerf_b200 import ops
    o, d = ol.random_rays(8192, seed=seed)
    bits = ol.sphere_bitfield(0.3, shell=0.03)[0]
    coords, _, ns, _ = ops.march(_cu(o), _cu(d), _cu(bits), (0.0, 1.0), 1 << 22, 0.00390625, 0.2, 5, True, ol.pcg32_seed(seed))
    cc, _, cnt = ops.compact(coords, ns, N_MAX)
    torch.cuda.synchronize()
    return cc, cnt[:1].clone()


def _trained():
    """coords, n_dev, grid and weights of one training step of a lego stand-in runner after 300 steps, as Runner.net_forward passes them"""
    from jnerf_b200 import ops
    from test_gpu_parity_e2e import _trained_runner
    r = _trained_runner("lego", 300)
    seen = {}
    orig = ops.network_fwd

    def spy(coords, grid, levels, wd, wr, n_dev=None, **kw):
        seen.update(coords=coords.clone(), n_dev=n_dev.clone(), grid=grid.detach().clone(), wd=wd.detach().clone(), wr=wr.detach().clone(),
                    lv=levels)
        return orig(coords, grid, levels, wd, wr, n_dev=n_dev, **kw)
    ops.network_fwd = spy
    try:
        r.train_step()
        torch.cuda.synchronize()
    finally:
        ops.network_fwd = orig
    return seen


# id -> (aabb, rows (int or a function of the SM count) or a source, regime)
CASES = {
    "lego-2^18": (1, N_MAX, "ref"),
    "fox-2^18": (4, N_MAX, "ref"),
    "march-2^18": (1, "march", "ref"),
    "rows-1": (1, 1, "ref"),
    "rows-127": (1, 127, "ref"),
    "rows-128": (1, 128, "ref"),
    "rows-129": (1, 129, "ref"),
    "one-tile-per-cta": (1, lambda sm: 2 * sm * ROWS, "ref"),
    "one-tile-per-cta+1": (1, lambda sm: 2 * sm * ROWS + 1, "ref"),
    "third-tile-one-row": (1, lambda sm: 4 * sm * ROWS + 1, "ref"),
    "rows-100003": (1, 100_003, "ref"),
    "tiny-grid": (1, N_MAX, "tiny"),
    "big-weights": (1, N_MAX, "big"),
    "trained-lego": (1, "trained", "trained"),
}


def _case(case):
    aabb, rows, regime = CASES[case]
    lv, cfg = _levels(aabb)
    seed = sum(map(ord, case))
    n_dev = None
    if regime == "trained":
        s = _trained()
        lv, coords, grid, wd, wr, n_dev = s["lv"], s["coords"], s["grid"], s["wd"], s["wr"], s["n_dev"]
        assert grid.numel() == cfg.n_params and lv.n_entries == cfg.n_entries
        return lv, cfg, coords, grid, wd, wr, n_dev
    n = rows(_sm()) if callable(rows) else (N_MAX if rows == "march" else rows)
    coords, grid, wd, wr, _ = ray_inputs(n, cfg.n_params, seed)
    if regime == "tiny":
        grid = (grid.astype(np.float32) * np.float32(1e-5)).astype(np.float16)         # encodings and densities are fp16 subnormals
    elif regime == "big":
        wd, wr = wd * np.float16(2), wr * np.float16(2)                                # each layer doubles: colour outputs grow 16-fold
    coords = _cu(coords)
    if rows == "march":
        coords, n_dev = _march_rows(seed)
    return lv, cfg, coords, _cu(grid), _cu(wd), _cu(wr), n_dev


@pytest.mark.parametrize("case", list(CASES))
def test_network_fwd_against_fp64(case):
    from jnerf_b200 import ops
    t0 = time.time()
    lv, cfg, coords, grid, wd, wr, n_dev = _case(case)
    n = coords.shape[0]
    nl = n if n_dev is None else min(int(n_dev.view(torch.int32)[0]), n)
    out, enc = _fwd(coords, grid, lv, wd, wr, n_dev)
    fails = []

    # the encoding: the oracle's, bit for bit, on both store paths; the per-row path gives the same outputs
    pos, dirs = coords[:nl, :3].cpu().numpy(), coords[:nl, 4:].cpu().numpy()
    with device_scales(lv):
        enc_ref = ol.hash_fwd(cfg, pos, grid.cpu().numpy(), acc32=True)
    bad = np.flatnonzero((enc[:nl].cpu().numpy().view(np.uint16) != enc_ref.view(np.uint16)).any(1))
    assert bad.size == 0, f"{bad.size} encoded rows differ from the oracle, first {bad[:8]}"
    out_b, enc_b = _fwd(coords, grid, lv, wd, wr, n_dev, off=4)
    assert torch.equal(_bits(out_b), _bits(out)), "the per-row store path changed the outputs"
    assert torch.equal(_bits(enc_b[:nl]), _bits(enc[:nl])), "the per-row store path saved another encoding"
    assert bool((_bits(out[nl:]) == SENTINEL).all()), "rows past the live count were written"
    out_c, enc_c = _fwd(coords, grid, lv, wd, wr, n_dev)
    assert torch.equal(_bits(out_c), _bits(out)) and torch.equal(_bits(enc_c), _bits(enc)), "repeated launches differ"

    # density_fwd: column 3, bit for bit
    sig = ops.density_fwd(coords[:nl, :3].contiguous(), grid, lv, wd)
    assert torch.equal(_bits(sig), _bits(out[:nl, 3])), f"{int((_bits(sig) != _bits(out[:nl, 3])).sum())} densities differ from column 3"

    # (a) interval, (b) per-tile agreement with the mirror
    sh_k = sh_f32(dirs).astype(np.float16)
    sh_lo, sh_hi = sh_interval(dirs)
    ch = interval_chain(enc[:nl], _cu(sh_k), sh_lo.cuda(), sh_hi.cuda(), wd, wr)
    got = out[:nl]
    inside, ratio = interval_check(got, ch)
    dens_inside, _ = interval_check(torch.cat([got[:, :3], sig[:, None]], 1), ch)
    if not bool(inside.all()):
        rows = torch.nonzero(~inside.all(1)).flatten()
        fails.append(f"{rows.numel()} rows outside the interval, first {rows[:8].tolist()}")
    if not bool(dens_inside[:, 3].all()):
        fails.append("density_fwd outside the h0 interval")
    share = tile_agreement(got, ch["out"])
    low = share.min(0).values if share.shape[0] else torch.ones(4, dtype=torch.float64)
    bad_tiles = torch.nonzero((share[:, :3] < RGB_FLOOR).any(1) | (share[:, 3] < DENSITY_FLOOR)).flatten()
    if bad_tiles.numel():
        fails.append(f"{bad_tiles.numel()} tiles below the agreement floors, first {bad_tiles[:8].tolist()}: {share[bad_tiles[:4]].tolist()}")
    rad = radius_ulps(ch)
    E = {k: float(v.max()) for k, v in ch["E"].items()}

    # routing probes: exact, every row
    enc64, sh64 = enc[:nl].to(torch.float64), _cu(sh_k).to(torch.float64)
    sh_o = ol.sh(dirs, np.float16)
    routed_sh = torch.zeros(nl, 16, dtype=torch.float64, device="cuda")
    for k0, srcs in probe_sets():
        pwd, pwr = (_cu(w) for w in probe_weights(k0, srcs))
        p_out, _ = _fwd(coords, grid, lv, pwd, pwr, n_dev)
        want = probe_expected(k0, srcs, enc64, sh64)
        g = p_out[:nl].to(torch.float64)
        miss = torch.nonzero((g != want).any(1)).flatten()
        if miss.numel():
            fails.append(f"probe {k0} {srcs}: {miss.numel()} rows routed wrongly, first {miss[:8].tolist()}: got {g[miss[:2]].tolist()}, "
                         f"want {want[miss[:2]].tolist()}")
        for i, (c, k) in enumerate(srcs):
            if k is None:
                routed_sh[:, c - 16] = g[:, i]
        if not bool((_bits(p_out[nl:]) == SENTINEL).all()):
            fails.append(f"probe {k0}: rows past the live count were written")
    lo, hi = sh_lo.cuda(), sh_hi.cuda()
    if not bool(((routed_sh >= lo) & (routed_sh <= hi)).all()):
        fails.append("routed SH features outside the float64 SH interval")
    oracle_sh_diff = int((routed_sh.cpu().numpy() != sh_o.astype(np.float64)).sum())

    fmt = lambda v: "[" + ", ".join(f"{float(x):.3g}" for x in v) + "]"
    print(f"[fwd-fp64] {case} n={n} live={nl}: worst interval ratio {fmt(ratio.max(0).values if nl else [0] * 4)}; "
          f"radius median / max rgb {float(rad[:, :3].median()) if nl else 0:.3g} / {float(rad[:, :3].max()) if nl else 0:.3g} ulp, "
          f"h0 {float(rad[:, 3].median()) if nl else 0:.3g} / {float(rad[:, 3].max()) if nl else 0:.3g} ulp; "
          f"lowest tile agreement {fmt(low)} over {share.shape[0]} tiles; "
          f"max E hd {E['hd']:.3g} h {E['h']:.3g} sh {E['sh']:.3g} h1 {E['h1']:.3g} h2 {E['h2']:.3g}; "
          f"routed SH != oracle SH on {oracle_sh_diff} of {nl * 16}; {time.time() - t0:.1f} s")
    assert not fails, fails[:6]


# ------------------------------------------------------------------------------------------------ live counts and store paths
def _live_ids():
    return ["0", "1", "333", "third-tile", "n_max", "n_max+5"]


def _live_value(key, sm):
    return {"0": 0, "1": 1, "333": 333, "third-tile": 4 * sm * ROWS + 77, "n_max": N_MAX, "n_max+5": N_MAX + 5}[key]


@pytest.mark.parametrize("live", _live_ids())
def test_rows_past_the_live_count(live):
    lv, cfg = _levels(1)
    coords, grid, wd, wr, _ = (_cu(a) for a in ray_inputs(N_MAX, cfg.n_params, 31))
    full, enc_full = _fwd(coords, grid, lv, wd, wr)
    v = _live_value(live, _sm())
    nl = min(v, N_MAX)
    end = min((nl + ROWS - 1) // ROWS * ROWS, N_MAX)                       # end of the last live tile
    n_dev = torch.tensor([v], dtype=torch.int32, device="cuda")
    written = {}
    for path, off in (("tma", 0), ("per-row", 4)):
        out, enc = _fwd(coords, grid, lv, wd, wr, n_dev, off=off)
        assert torch.equal(_bits(out[:nl]), _bits(full[:nl])), f"{path}: live rows differ from a launch without a live count"
        assert torch.equal(_bits(enc[:nl]), _bits(enc_full[:nl])), f"{path}: live encoded rows differ"
        assert bool((_bits(out[nl:]) == SENTINEL).all()), f"{path}: out rows at or past n_dev were written"
        assert bool((_bits(enc[end:]) == SENTINEL).all()), f"{path}: enc rows past the last live tile were written"
        tail = (_bits(enc[nl:end]) != SENTINEL).any(1)
        written[path] = int(tail.sum())
        if path == "per-row":
            assert written[path] == 0, "the per-row path wrote enc rows of the last live tile past n_dev"
    print(f"[fwd-live] n_dev={v}: last live tile ends at {end}; enc rows written past n_dev: {written}")


def test_render_call_shape():
    """What render_rays does: out a view into a uint8 workspace, save_enc=False, n_dev read from the same workspace and far below n_max"""
    from jnerf_b200 import ops
    lv, cfg = _levels(1)
    coords, grid, wd, wr, _ = ray_inputs(N_MAX, cfg.n_params, 41)
    cap = N_MAX
    nbytes, off_rows, off_net, off_cnt = ops.render_workspace_layout(1000, cap)
    ws = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda")
    rows = ws[off_rows:off_rows + 28 * cap].view(torch.float32).view(cap, 7)
    rows.copy_(_cu(coords))
    out_rows = ws[off_net:off_net + 8 * cap].view(torch.float16).view(cap, 4)
    n_rows = ws[off_cnt:off_cnt + 4].view(torch.int32)
    n_rows.fill_(5003)
    before = ws.clone()
    ops.network_fwd(rows, _cu(grid), lv, _cu(wd), _cu(wr), n_dev=n_rows, save_enc=False, out=out_rows)
    torch.cuda.synchronize()
    ref, _ = _fwd(_cu(coords), _cu(grid), lv, _cu(wd), _cu(wr))
    assert torch.equal(_bits(out_rows[:5003]), _bits(ref[:5003]))
    changed = torch.nonzero(ws != before).flatten()
    assert changed.numel() == 0 or (int(changed.min()) >= off_net and int(changed.max()) < off_net + 8 * 5003), "bytes outside the live rows changed"


# ------------------------------------------------------------------------------------------------ lattice
def test_density_lattice_against_density_fwd():
    """n = 97: 912 673 rows, 7131 tiles (more than four per CTA), the last one 33 rows.  Woutd row 0 is scaled by 2048 so that the
    densities reach the hundreds and thousands, where the truncation keeps most fp16 bits and a one-ulp change of a position shows."""
    from jnerf_b200 import ops
    lv, cfg = _levels(1)
    _, grid, wd, _, _ = ray_inputs(1, cfg.n_params, 51)
    wd = wd.copy()
    wd[2048:2048 + 64] = (wd[2048:2048 + 64].astype(np.float32) * 2048).astype(np.float16)
    n = 97
    assert n ** 3 // ROWS > 4 * _sm() and n ** 3 % ROWS
    field = ops.density_lattice(n, _cu(grid), lv, _cu(wd))
    q = np.arange(n, dtype=np.float32) / np.float32(n - 1)
    pos = np.stack(np.meshgrid(q, q, q, indexing="ij"), -1).reshape(-1, 3)
    sig = ops.density_fwd(_cu(pos), _cu(grid), lv, _cu(wd)).float()
    want = torch.trunc(sig.clamp_min(0))
    got = field.reshape(-1)
    bad = torch.nonzero(got.view(torch.int32) != want.view(torch.int32)).flatten()
    print(f"[fwd-lattice] n={n}: share of densities above 128 {float((sig > 128).double().mean()):.3f}")
    assert bad.numel() == 0, f"{bad.numel()} lattice values differ, first {bad[:8].tolist()}"
