"""The fused NGP backward (network_bwd256_kernel, through ngp_network_bwd_fx) against fp64 references at training batch sizes, with
error bounds that hold for any summation order the kernel may choose and fail for a wrong gradient.

Two weight sets per case:
- probe: the density net passes the output gradient straight through.  W0d row j is e_j and row 32 + j is -e_j, Woutd row 0 is
  [+1] * 32 + [-1] * 32 and its other rows are zero, and the colour net's first 16 input columns (the density features) are zero.
  Then hd = [relu(enc) | relu(-enc)], dYd = [dsig, 0, ...], and d_enc[r, k] = dsig[r] where enc[r, k] != 0 and 0 where it is zero:
  every value on the way is an exact fp16, so the hash-grid gradient reference needs no allowance for rounding upstream of the
  scatter.  The colour net still runs on the SH features and has weight gradients.
- realistic: random weights and an O(1) grid.  The reference is a float64 chain started from the kernel's own encoded rows that
  rounds to fp16 wherever the kernel stores to a shared-memory slab, so it differs from the kernel only where an fp32 sum lies next
  to an fp16 rounding boundary (a "flip").

Hash-grid gradient.  The scatter sums the contributions dy * w of a run of at most B3_RUN consecutive rows of one level that stay in
one grid cell in an fp32 register, one fmaf per row, then adds round(2^32 * sum) to a 64-bit integer.  Per feature of entry e, with
g_e the exact sum of its contributions, A_e the sum of their magnitudes and cnt_e their number (oracle orc_hash_bwd_f64):
- a run of k <= B3_RUN terms rounds k times (the first fmaf already rounds the product), each time by at most u = 2^-24 of a partial
  sum, so its fp32 sum is off by at most gamma_k * (sum of its |terms|), gamma_k = k u / (1 - k u) (Higham, Accuracy and Stability of
  Numerical Algorithms, 2nd ed., section 4.2); summed over the runs that reach e this is at most gamma_B3_RUN * A_e;
- each run is rounded to the nearest multiple of 2^-32 once, off by at most 2^-33, and at most cnt_e runs reach e (a run of zero
  terms adds nothing);
- the integer sums are exact, the clamp to +-65504 never acts on these inputs, and fx * 2^-32 is exact in float64.
So |fx_e 2^-32 - g_e| <= gamma_B3_RUN A_e + cnt_e 2^-33, whatever the order of the runs and of the rows among runs; an entry with
cnt_e = 0 must hold exactly 0.  The probe tier holds every entry to this.  A single contribution below 2^-32 uses all of the second
term, so the worst ratio of error to bound is close to 1 by construction.  In the realistic tier a flip upstream moves d_enc by up
to a few ulps of the terms it is summed from, which can be many ulps of d_enc itself where they cancel.  So each entry also gets
2^-6 A'_e, A'_e being the scatter of sum_o |g_hd[o] W0d[o, k]|.  Up to 2e-4 of the touched entries may fall outside that, and the
normwise error is held to 4e-3.  On an H100 the worst observed values were 2.6e-5 and 8.5e-4, with about 1e-4 of entries outside
the fp32 bound plus 2^-10 A'_e.

Weight gradients.  Each CTA sums the products of its rows in fp32 tensor-core accumulators, at most 8 pairs = 2048 rows at 2^18 rows
on 132 SMs, and the test adds the CTAs' slots in float64.  Recursive fp32 summation of 2048 terms is off by at most 2048 * 2^-24 =
2^-13 of the sum of their magnitudes; the bound allows 2^-12 for accumulators that truncate instead of rounding to nearest.  That
holds for the probe's density net, whose operands are exact: the observed worst is 6e-4 of the bound.  The mirror reproduces the
colour net (both tiers) and the realistic density net only up to flips, and rows that repeat (the adversarial case has blocks of
512 identical rows) repeat a flip.  Those gradients are held to 2^-6 of the sum of |term|; the observed worst is 2^-8.7.

The forward's saved encoding, which the backward loads by TMA, must equal the oracle's fp32-accumulated encoding bit for bit.

Level tables stay alive in _TABLES (ngp_network_bwd keys its own scratch on a table's address; ngp_network_bwd_fx uses caller-owned
scratch and cannot hit that)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

import oracle_lib as ol
from ngp_fwd_ref import WD_N, WR_N, mirror
from test_gpu_ops import device_scales

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_bwd_digests import inputs as ray_inputs  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _b3_run():
    """The longest run the scatter sums in one fp32 register: the 256 rows of a pair split into B3_RUNS runs (fused_net.cu)."""
    src = open(os.path.join(ROOT, "jnerf_b200", "csrc", "fused_net.cu")).read()
    runs = int(re.search(r"\bB3_RUNS = (\d+)", src).group(1))
    return -(-256 // runs)


B3_RUN = _b3_run()
U32 = 2.0 ** -24
GAMMA = B3_RUN * U32 / (1 - B3_RUN * U32)
W_REL = 2.0 ** -12
W_FLIP = 2.0 ** -6          # weight gradients whose operands the mirror reproduces only up to flips (observed: at most 2^-8.7)
FLIP_GRID = 2.0 ** -6       # realistic tier, per entry: flips of d_enc, relative to the scatter of its terms' magnitudes
GRID_OUTLIERS = 2e-4        # realistic tier: share of touched entries allowed outside bound + flips (observed: at most 2.6e-5)
GRID_NORM = 4e-3            # realistic tier: normwise error of the hash-grid gradient (observed: at most 8.5e-4)

_TABLES = {}


def _levels(aabb, log2T):
    from jnerf_b200 import ops
    if (aabb, log2T) not in _TABLES:
        _TABLES[(aabb, log2T)] = (ops.HashLevels(aabb, log2_hashmap_size=log2T), ol.HashCfg(aabb, log2_hashmap_size=log2T))
    return _TABLES[(aabb, log2T)]


def test_mirror_matches_oracle_mlp():
    """The float64 mirror against the oracle's fp32 MLP (orc_mlp_fwd / orc_mlp_bwd) at n = 3000.  Each side feeds a layer its own
    rounded inputs, so one-ulp flips propagate down the chain (and the oracle side rounds dYd twice); a transposed weight, a wrong mask
    or a misplaced column changes most values instead.  The first layer, from identical inputs, must agree to one ulp everywhere; every
    stage to 1e-3 normwise with at most 5 % of its values beyond one ulp (observed: 2e-4 and 2.7 % at d_enc, the end of the chain);
    the weight gradients within the bound the kernel is held to."""
    n = 3000
    coords, grid, wd, wr, dout = ray_inputs(n, 2 * 4096, 7)
    rng = np.random.default_rng(7)
    enc = rng.uniform(-1, 1, (n, 32)).astype(np.float16)
    sh = ol.sh(coords[:, 4:].copy(), np.float16)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out, s, d_enc, (dwd, awd), (dwr, awr) = mirror(t(enc), t(sh), t(dout), t(wd), t(wr))
    h, inter_d = ol.mlp_fwd(wd, enc, 0)
    rin = np.concatenate([h, sh], 1)
    r, inter_r = ol.mlp_fwd(wr, rin, 1)
    dYr = np.zeros((n, 16), np.float16)
    dYr[:, :3] = dout[:, :3]
    d_rin, temps_r, dWr = ol.mlp_bwd(wr, rin, inter_r, dYr, 1, 3)
    dYd = (d_rin[:, :16].astype(np.float32) + np.pad(dout[:, 3:].astype(np.float32), ((0, 0), (0, 15)))).astype(np.float16)
    d_enc_o, temps_d, dWd = ol.mlp_bwd(wd, enc, inter_d, dYd, 0, 16)

    def close16(mine, theirs, name):
        a, b = mine.cpu().numpy().astype(np.float64), np.asarray(theirs, np.float64)
        ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float16)).astype(np.float64)
        d = np.abs(a - b)
        if name == "hd":
            assert (d <= ulp).all(), name
        assert np.linalg.norm(d) <= 1e-3 * np.linalg.norm(b), (name, np.linalg.norm(d) / np.linalg.norm(b))
        assert (d > ulp).mean() <= 0.05, (name, (d > ulp).mean())

    close16(s["hd"], inter_d, "hd")
    close16(s["h"], h, "h")
    close16(s["h1"], inter_r[:n], "h1")
    close16(s["h2"], inter_r[n:], "h2")
    close16(out[:, :3], r[:, :3], "rgb")
    close16(s["g_h2"], temps_r[:n], "g_h2")
    close16(s["g_h1"], temps_r[n:], "g_h1")
    close16(s["dYd"], dYd, "dYd")
    close16(s["g_hd"], temps_d, "g_hd")
    close16(d_enc, d_enc_o, "d_enc")
    for got, ab, want in ((dwd, awd, dWd), (dwr, awr, dWr)):
        assert (np.abs(got.cpu().numpy() - want) <= W_REL * ab.cpu().numpy()).all()


# ------------------------------------------------------------------------------------------------ cases
# id -> (aabb, log2 T, rows launched, live rows on the device or None, seed)
CASES = {
    "lego": (1, 19, 1 << 18, None, 101),
    "fox-live": (4, 19, 1 << 18, 200_001, 102),
    "odd": (1, 19, 100_003, None, 103),
    "cfg1": (1, 14, 1 << 18, None, 104),                     # 2^14 entries per level: heavy hash collisions
    "one-extra-pair": (1, 19, "sm+", None, 105),            # 256 * sm_count + 129 rows: CTA 0 walks two pairs, the last tile B has one row
    "tiny-1": (1, 19, 1, None, 106),
    "tiny-127": (1, 19, 127, None, 107),
    "tiny-129": (1, 19, 129, None, 108),
    "adversarial": (4, 19, 65_536, None, 109),
}


def _adversarial_coords(n, rng):
    """Blocks of 256 and 512 identical rows, coordinates exactly 0.0 and 1.0, coordinates on and next to level-0 cell faces
    (x * 15 + 0.5 an integer), and 64-row segments that step only in z."""
    x = rng.random((n, 3), dtype=np.float32)
    faces = np.float32((np.arange(1, 16) - 0.5) / 15)
    faces = np.concatenate([faces, np.nextafter(faces, np.float32(0)), np.nextafter(faces, np.float32(1)), np.float32([0, 1])])
    b = 0
    for blk, size in enumerate([512, 256, 256, 512, 256]):                    # identical rows
        x[b:b + size] = [rng.random(3, dtype=np.float32), [0, 0, 0], [1, 1, 1], [0, 1, 0.5], faces[[3, 20, 40]]][blk]
        b += size
    seg = b
    while seg + 64 <= n // 2:                                                  # z-only segments, some starting on a face
        z0 = rng.choice(faces) if rng.random() < 0.5 else rng.random(dtype=np.float32)
        x[seg:seg + 64, :2] = rng.random(2, dtype=np.float32)
        x[seg:seg + 64, 2] = np.clip(z0 + np.float32(0.003) * np.arange(64, dtype=np.float32), 0, 1)
        seg += 64
    rest = slice(n // 2, n)                                                    # random rows, components snapped to 0, 1 or a face
    m = rng.random((n - n // 2, 3))
    x[rest] = np.where(m < 0.1, np.float32(0), np.where(m < 0.2, np.float32(1), np.where(m < 0.4, rng.choice(faces, (n - n // 2, 3)), x[rest])))
    return x


def _probe_weights(wd, wr):
    wd, wr = wd.copy(), wr.copy()
    w0d = np.zeros((64, 32), np.float16)
    w0d[np.arange(32), np.arange(32)] = 1
    w0d[32 + np.arange(32), np.arange(32)] = -1
    woutd = np.zeros((16, 64), np.float16)
    woutd[0] = [1] * 32 + [-1] * 32
    wd[:] = np.concatenate([w0d.ravel(), woutd.ravel()])
    wr[:2048].reshape(64, 32)[:, :16] = 0
    return wd, wr


def _run(case, tier):
    from jnerf_b200 import ops
    aabb, log2T, n, live, seed = CASES[case]
    sm = int(ops.lib.load().ngp_sm_count())
    if n == "sm+":
        n = 256 * sm + 129
    lv, cfg = _levels(aabb, log2T)
    coords, grid, wd, wr, dout = ray_inputs(n, cfg.n_params, seed)
    rows = min(n, 5)                                         # the inputs' zero-gradient runs start at row 0: the tiny cases need gradients
    dout[:rows] = (np.random.default_rng(seed).standard_normal((rows, 4)) * 0.05).astype(np.float16)
    if case == "adversarial":
        coords[:, :3] = _adversarial_coords(n, np.random.default_rng(seed))
    if tier == "probe":
        wd, wr = _probe_weights(wd, wr)
    nl = n if live is None else live
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    n_dev = None if live is None else torch.tensor([live], dtype=torch.int32, device="cuda")
    ct, wdt, wrt, dt = t(coords), t(wd), t(wr), t(dout)
    out, enc = ops.network_fwd(ct, t(grid), lv, wdt, wrt, n_dev=n_dev)
    fx, part = ops.network_bwd_scratch(lv)
    ops.network_bwd_fx(ct, enc, lv, wdt, wrt, dt, fx, part, n_dev=n_dev)
    torch.cuda.synchronize()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    pos = coords[:nl, :3].copy()
    return dict(n=n, nl=nl, sm=sm, cfg=cfg, lv=lv, pos=pos, coords=coords, grid=grid, dout=dout, wd=wd, wr=wr,
                out=out[:nl], enc=enc[:nl], fx=fx, part=part)


@pytest.mark.parametrize("tier", ["probe", "realistic"])
@pytest.mark.parametrize("case", list(CASES))
def test_network_bwd_against_fp64(case, tier):
    r = _run(case, tier)
    n, nl, cfg, lv, pos = r["n"], r["nl"], r["cfg"], r["lv"], r["pos"]
    enc = r["enc"]
    report = [f"{case}/{tier} n={n} live={nl}"]
    fails = []

    # forward: the saved encoding is the oracle's, bit for bit (this is what the backward's TMA load reads)
    with device_scales(lv):
        enc_ref = ol.hash_fwd(cfg, pos, r["grid"], acc32=True)
    enc_np = enc.cpu().numpy()
    bad = np.flatnonzero((enc_np.view(np.uint16) != enc_ref.view(np.uint16)).any(1))
    assert bad.size == 0, f"{bad.size} encoded rows differ from the oracle, first {bad[:8]}"

    # the float64 mirror, started from the kernel's own encoding
    sh = torch.from_numpy(ol.sh(r["coords"][:nl, 4:].copy(), np.float16)).cuda()
    dout = torch.from_numpy(r["dout"][:nl]).cuda()
    out_ref, slabs, d_enc, (gwd, awd), (gwr, awr) = mirror(enc, sh, dout, torch.from_numpy(r["wd"]).cuda(), torch.from_numpy(r["wr"]).cuda())
    if tier == "probe":
        d_probe = torch.where(enc != 0, dout[:, 3:4], torch.zeros_like(dout[:, 3:4])).to(torch.float64)
        assert torch.equal(d_enc, d_probe), "the probe weights must pass dL/dsigma straight to every nonzero feature"

    # forward output: within 2 fp16 ulps of max(|ref|, 1) on at least 99.9 % of the rows
    ulp = torch.exp2(torch.floor(torch.log2(out_ref.abs().clamp_min(1.0))) - 10)
    row_ok = ((r["out"].to(torch.float64) - out_ref).abs() <= 2 * ulp).all(1)
    assert row_ok.double().mean() >= 0.999, float(row_ok.double().mean())
    report.append(f"out rows within 2 ulp {float(row_ok.double().mean()):.6f}")

    # hash-grid gradient against the exact scatter of the reference d_enc
    with device_scales(lv):
        g, a, cnt = ol.hash_bwd_f64(cfg, pos, d_enc.to(torch.float32).cpu().numpy())
    got = r["fx"].cpu().numpy().astype(np.float64) * 2.0 ** -32
    err = np.abs(got - g)
    bound = GAMMA * a + cnt * 2.0 ** -33
    touched = cnt > 0
    assert touched.any()
    if tier == "probe":
        assert (got[~touched] == 0).all(), f"{int((got[~touched] != 0).sum())} entries without a contribution were written"
        over = np.flatnonzero(err > bound)
        assert over.size == 0, f"{over.size} entries outside the bound, first {over[:8]}: got {got[over[:4]]}, want {g[over[:4]]}"
        report.append(f"grid worst err/bound {np.max(err[touched] / bound[touched]):.3g}")
    else:
        with device_scales(lv):
            a_in, _, _ = ol.hash_bwd_f64(cfg, pos, slabs["d_enc_abs"].to(torch.float32).cpu().numpy())
        nt = int(touched.sum())
        allow = bound + FLIP_GRID * a_in
        n_out = int((err > allow).sum())
        norm = np.linalg.norm(got - g) / max(np.linalg.norm(g), 1e-300)
        report.append(f"grid outside bound + flips {n_out}/{nt}, outside the fp32 bound alone {int((err > bound).sum())}, normwise {norm:.3g}")
        if n_out > GRID_OUTLIERS * nt:
            fails.append(f"{n_out} of {nt} touched entries outside the bound")
        if norm > GRID_NORM:
            fails.append(f"normwise {norm}")

    # weight gradients: the CTAs' slots in float64 against the mirror
    slots = min(((n + 127) // 128 + 1) // 2, r["sm"])         # bwd_ctas(n): the slots of later CTAs are stale
    s = r["part"].view(-1, WD_N + WR_N)[:slots].to(torch.float64).sum(0)
    for name, got_w, want, ab in (("density", s[:WD_N], gwd, awd), ("colour", s[WD_N:], gwr, awr)):
        rel = W_REL if (tier, name) == ("probe", "density") else W_FLIP      # exact operands only in the probe's density net
        e = (got_w - want).abs()
        bad = torch.nonzero(e > rel * ab).flatten()
        if bad.numel():
            fails.append(f"{name} weight gradient: {bad.numel()} elements outside the bound, first {bad[:8].tolist()}")
        nz = ab > 0
        report.append(f"{name} weights worst err/sum|term| {float((e[nz] / ab[nz]).max()) if nz.any() else 0.0:.3g} (bound {rel:.3g})")
    if not torch.equal(s[WD_N + 6144 + 3 * 64:], torch.zeros_like(s[WD_N + 6144 + 3 * 64:])):
        fails.append("colour Wout rows >= 3 must stay zero")
    print("[bwd-fp64] " + "; ".join(report))
    assert not fails, fails
