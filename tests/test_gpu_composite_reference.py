"""The NGP composite kernels (ngp_composite_fwd / _infer / _bwd and the fused training tail ngp_composite_loss_bwd, sampler.cu) against
a float64 composite (oracle orc_composite_f64) at training batch sizes, with an error bound for every colour, alpha, loss and dL/dnet
entry; and the march and compaction bookkeeping at those sizes against the oracle, bit for bit.

Error bound.  u = 2^-24.  Every fp32 operation is modelled by its documented error, and the oracle carries an (exact value, bound)
pair through the kernel's expression tree in the kernel's association order wherever that order is fixed:
- a rounded multiply or add of inputs a, b with errors ea, eb: |a| eb + |b| ea + ea eb for the inputs, u (|v| + e) for the
  rounding, and 2^-150 for a result in the subnormal range (the kernels do not flush fp32 subnormals);
- __expf(x): (2 + floor(1.173 |x|)) ulp (CUDA Programming Guide, intrinsic functions), an ulp being at most 2^-23 of the result,
  plus 2^-126 for a result the special-function unit flushes to zero.  It enters the density exp(o_w), the transmittance factor
  exp(-sigma dt) and the clamped density derivative exp(clamp(o_w, -15, 15));
- logistic_sfu(x) = __fdividef(1, 1 + __expf(-x)): the __expf error, one rounded add, and __fdividef's 2 ulp (4u) for denominators
  in [2^-126, 2^126]; beyond 2^126 it returns 0, an absolute error below 2^-126.  With E = e^-x and c = 1 / (1 + E) this gives
  |c~ - c| <= c ((1 + 4u) / ((1 - (1 - c) e_x) (1 - u)) - 1) + 2^-126, relative to c: a saturated colour is accurate in absolute
  terms only, and the c (1 - c) of the colour gradient is held to an absolute bound;
- alpha: the kernel's exp(fl(-fl(__expf(o_w)) dt)) is bracketed by evaluating exp at the extremes of its argument (not a first-order
  estimate, so it holds for any o_w: an infinite density gives alpha = 1 exactly); alpha = fl(1 - E2) and the factor fl(1 - alpha)
  each add u of their value.  These are absolute errors of about u: a nearly transparent sample's alpha is relatively inaccurate;
- transmittance T_j = prod_{k<j} (1 - alpha_k): the exact product of the factors at their upper and lower bounds brackets the product
  of the kernel's factors, and the j - 1 roundings of the product add gamma_j = j u / (1 - j u) of it, plus j 2^-150.  This holds
  for ANY association, so it covers the COMP_K-sample lane products, the 32-lane scan, the carries across 128-sample chunks, the
  backward's separate recomputation in another order, and the oracle's serial loop alike;
- colour sums (forward colour, the backward's running colour `run`): m fmaf terms w_k c_k in any binary tree round at most m times
  on the way from a term to the result (every rounding node has a non-zero sibling subtree), so the error is gamma_m sum |w_k c_k|
  plus the propagated errors of the terms.  Again association-free: this does not read the tree depth from the kernel;
- the background fmaf(T, bg, rgb) is one more term; the suffix rr - run is a rounded subtraction of an exact rr (the kernel's own
  forward colour) from run, so its bound is ABSOLUTE, of the size of run's bound, however much cancels; the three-term dot product
  is evaluated as Eigen's x0 + (x1 + x2); then the products by dd, dt and loss_scale (the kernels' fp32 128 / R), and the l1 term
  -1e-4 * reg_scale for o_w < 0.  dt is the kernel's own fp32 value (nerf_unwarp_dt is one fmaf), so it carries no error.
These are the first-order expansions of exact identities except where stated; SAFETY = 2 covers the second-order remainder.

fp16 dL/dnet: the kernel stores rn16(d~) for an fp32 d~ within the bound of the exact d.  rn16 is monotone, so that is exactly
rn16(d - S e) <= h <= rn16(d + S e): a correctly rounded value, with the fp16 subnormal spacing 2^-24 below 2^-14 and +-inf at and
above 65520; a zero only where the interval reaches zero.  A store that flushed subnormals to zero fails this.

The loss: loss_out must equal the Huber sum of the kernel's own colour, branch by branch as the kernel's fp32 expression takes it
(numpy float32 reproduces `rel > delta` and diff / delta exactly), within the rounding of its fp32 operations.

The backward is checked against its own upstream values: rr is the kernel's forward colour and lg the fp32 Huber gradient of it,
so a forward error does not leak into the backward's bound.  The bound is rehearsed on the oracle's serial fp32 composite in
test_composite_bound_cpu.py.

Findings on an H100 80GB HBM3 (700 W power limit), the whole file in 33 s:
- the fused tail and the unfused pair agree bit for bit (the same inlined composite_ray_fwd / _bwd, sampler.cu built -fmad=false);
- worst ratio of error to bound over all cases: forward colour 0.16, inference colour 0.17, alpha 0.25, loss 0.31, fp32 dL/dnet
  colour 0.48 and density 0.30.  An fp16 entry's ratio includes half an fp16 ulp and is close to 1 by construction;
- at training size 81-90 % of the non-zero fp16 dL/dnet entries are fp16 subnormals (89 % in a lego step after 100 training steps),
  and the kernel rounds them correctly: the store does not flush them."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

import oracle_lib as ol

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_llff_cpu import shells_bitfield, wide_rays  # noqa: E402

pytestmark = pytest.mark.gpu

SAFETY = 2.0
DELTA = 0.1
CAP = 1 << 18                       # the compaction cap of a training step (sampler.target_batch_size)
MAX_SAMPLES = 1 << 22               # the march's raw capacity here (ol.march allocates MAX_SAMPLES x 7 floats on the host)
EDGE_LENGTHS = [0, 1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024]
SENTINEL = np.float16(-1234.0)


# ------------------------------------------------------------------------------------------------ bound checks (shared with the CPU rehearsal)
def l1_of(mean, reg_scale=1.0):
    """The kernels' density regulariser: (mean < 0.01f ? 1e-4f : 0) * reg_scale, in fp32."""
    return np.float32(1e-4 if np.float32(mean) < np.float32(0.01) else 0.0) * np.float32(reg_scale)


def huber_f32(rgb, target, delta=DELTA):
    """huber_loss.py:11-14 as the fused kernel evaluates it in fp32: (lg, big) with big = rel > delta."""
    r, t, d = np.asarray(rgb, np.float32), np.asarray(target, np.float32), np.float32(delta)
    diff = r - t
    rel = np.abs(diff)
    big = rel > d
    lg = np.where(big, np.where(diff > 0, np.float32(1), np.float32(-1)), diff / d).astype(np.float32)
    return lg, big


def _ev_round(v, e):
    return v, e + 2.0 ** -24 * (np.abs(v) + e) + 2.0 ** -150


def loss_bound(rgb, target, delta=DELTA):
    """Exact Huber sum (float64) of the kernel's own fp32 colour, on the kernel's branches, and its error bound."""
    _, big = huber_f32(rgb, target, delta)
    d = np.float32(delta)
    dv, de = _ev_round(np.asarray(rgb, np.float64) - np.asarray(target, np.float32).astype(np.float64), 0.0)
    rel = np.abs(dv)
    lv_big, le_big = _ev_round(rel - np.float64(np.float32(0.5) * d), de)
    h = np.float64(np.float32(0.5) / d)
    mv, me = _ev_round(h * rel, h * de)
    sv, se = _ev_round(mv * rel, mv * de + rel * me + me * de)
    lv, le = np.where(big, lv_big, sv), np.where(big, le_big, se)
    tv, te = lv[:, 0], le[:, 0]
    for k in (1, 2):
        tv, te = _ev_round(tv + lv[:, k], te + le[:, k])
    return tv, te


def ratio32(got, exact, err):
    """|got - exact| / (SAFETY err); an entry with a zero bound must be exact."""
    d = np.abs(np.asarray(got, np.float64) - exact)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, d / (SAFETY * err), np.where(d == 0, 0.0, np.inf))
    return np.where(np.isnan(d), np.inf, r)


def check16(got, exact, err):
    """(ok, ratio): ok where the fp16 value is a correct rounding of a value within SAFETY err of exact; ratio = |got - exact| over
    (SAFETY err + half the fp16 spacing at exact), for the report."""
    with np.errstate(over="ignore", invalid="ignore"):
        lo = (exact - SAFETY * err).astype(np.float16).astype(np.float64)
        hi = (exact + SAFETY * err).astype(np.float16).astype(np.float64)
        g = np.asarray(got).astype(np.float64)
        ok = (g >= lo) & (g <= hi)
        sp = np.spacing(np.abs(exact).astype(np.float16)).astype(np.float64)
        r = np.abs(g - exact) / (SAFETY * err + 0.5 * sp)
    return ok, np.where(ok, np.nan_to_num(r, nan=0.0, posinf=0.0), np.inf)


def covered(ns_c, n_rows):
    m = np.zeros(n_rows, bool)
    for n, b in np.asarray(ns_c).view(np.uint32).reshape(-1, 2):
        m[b:b + n] = True
    return m


def check_dnet(got, ex, cov, stats, tag, fails):
    """Every covered dL/dnet entry within its bound.  stats: worst ratio per dtype for colour and density entries; for fp16 also the
    worst ratio over the entries whose exact value is an fp16 subnormal, their share among the non-zero entries, and the smallest
    share of entries that equal the exact value correctly rounded."""
    x, e = ex["dnet"][cov], ex["dnet_err"][cov]
    g = np.asarray(got)[cov]
    if g.size == 0:
        return
    if g.dtype == np.float16:
        ok, r = check16(g, x, e)
        sub = (np.abs(x) > 0) & (np.abs(x) < 2.0 ** -14)
        if sub.any():
            note(stats, "dnet fp16 subnormal", r[sub].max())
            note(stats, "subnormal share", sub.sum() / max(1, (x != 0).sum()))
        with np.errstate(over="ignore"):
            same = float((g.view(np.uint16) == x.astype(np.float16).view(np.uint16)).mean())
        stats["fp16 = rn16(exact) share"] = min(stats.get("fp16 = rn16(exact) share", 1.0), same)
    else:
        r = ratio32(g, x, e)
        ok = r <= 1
    dn = np.dtype(g.dtype).name
    note(stats, f"dnet colour {dn}", r[:, :3].max())
    note(stats, f"dnet density {dn}", r[:, 3].max())
    if not ok.all():
        bad = np.argwhere(~ok)
        i, k = bad[0]
        fails.append(f"{tag}: {len(bad)} dnet entries outside the bound, first row {np.flatnonzero(cov)[i]} col {k}: "
                     f"got {g[i, k]!r}, exact {x[i, k]!r}, bound {SAFETY * e[i, k]!r}")


def check_rays(got, exact, err, stats, name, tag, fails):
    r = ratio32(got, exact, err)
    note(stats, name, r.max() if r.size else 0.0)
    if not (r <= 1).all():
        i = np.unravel_index(np.argmax(r), r.shape)
        fails.append(f"{tag}: {int((r > 1).sum())} {name} entries outside the bound, worst at {i}: got {np.asarray(got)[i]!r}, "
                     f"exact {exact[i]!r}, bound {SAFETY * err[i]!r}")


def note(stats, key, v):
    stats[key] = max(stats.get(key, 0.0), float(v))


# ------------------------------------------------------------------------------------------------ synthetic ray batches
TAUS = [0.05, 0.7, 3.0, 9.5, 14.0]     # optical depth of a whole ray: 9.5 and 14 leave T ~ 7e-5 and 8e-7 in front of the background
ADV_DENSITY = np.float32([15, -15, 15.0078125, 14.9921875, -15.0078125, -14.9921875, 14.5, 14.6, -14.6, 0, 0, 0, -30, -1000, 50, 100, 65504])
ADV_COLOUR = np.float32([17, -17, 17.5, -17.5, 20, -20, 100, -100, 0, 16.9, -16.9, 65504, -65504])


def lengths_batch(lengths, seed, cut_share=0.2, gaps=True, adversarial=False, opaque=True):
    """Rows of rays with the given sample counts: (net fp32 values, coords, numsteps_in, numsteps_c, bg, target).  Ray i's density
    gives it a total optical depth TAUS[i % 5]; some rays turn opaque (o_w = 40) in their first, middle or last chunk; cut_share of the
    rays are cut (numsteps_in > numsteps_c: no background); with gaps, compacted bases leave unused rows between rays."""
    rng = np.random.default_rng(seed)
    R = len(lengths)
    n = np.asarray(lengths, np.int64)
    gap = rng.integers(0, 3, R) if gaps else np.zeros(R, np.int64)
    base = np.concatenate([[0], np.cumsum(n + gap)[:-1]]) + gap
    S = int((base + n).max()) + 3 if R else 3
    coords = rng.random((S, 7), dtype=np.float32)
    net = np.zeros((S, 4), np.float32)
    net[:, :3] = rng.normal(0, 2.5, (S, 3))
    mn, mx = np.sqrt(3.0) / 1024, np.sqrt(3.0) / 1024 * 16
    for i in range(R):
        if n[i] == 0:
            continue
        rows = slice(base[i], base[i] + n[i])
        dt = coords[rows, 3].astype(np.float64) * (mx - mn) + mn
        net[rows, 3] = np.log(TAUS[i % 5] / (n[i] * dt)) + rng.normal(0, 0.3, n[i])
        if opaque and i % 7 == 3:
            chunk = [0, (n[i] - 1) // 256 * 128, (n[i] - 1) // 128 * 128][(i // 7) % 3]
            net[base[i] + min(n[i] - 1, chunk + int(rng.integers(0, 128))), 3] = 40
        if adversarial:
            pick = rng.random(n[i]) < 0.08
            net[rows, 3][pick] = rng.choice(ADV_DENSITY, int(pick.sum()))
            pick = rng.random((n[i], 3)) < 0.1
            net[rows, :3][pick] = rng.choice(ADV_COLOUR, int(pick.sum()))
    ns_c = np.stack([n, base], 1).astype(np.int32)
    ns_in = ns_c.copy()
    cut = (rng.random(R) < cut_share) & (n > 0)
    ns_in[cut, 0] += rng.integers(1, 50, int(cut.sum()))
    bg = rng.random((R, 3), dtype=np.float32)
    target = rng.random((R, 3), dtype=np.float32)
    return dict(net=net, coords=coords, ns_in=ns_in, ns_c=ns_c, bg=bg, target=target, cascades=5, mean=0.001)


def edge_batches():
    out = [lengths_batch([n], seed=100 + n, cut_share=0.0, gaps=False) for n in EDGE_LENGTHS]
    for r in range(1, 8):
        R = 16 + r
        out.append(lengths_batch(list(np.resize(np.roll(EDGE_LENGTHS, r), R)), seed=200 + r))
    return out


def adversarial_batch(seed=300):
    rng = np.random.default_rng(seed)
    lengths = list(rng.integers(1, 300, 58)) + [1024, 700, 129]
    b = lengths_batch(lengths, seed, adversarial=True)
    b["rr_offset"] = 0.25            # a second backward with rr = rgb + 0.25: makes samples behind an opaque one carry a gradient
    return b


# ------------------------------------------------------------------------------------------------ GPU side
def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _twice(fn):
    a, b = fn(), fn()
    ta = a if isinstance(a, tuple) else (a,)
    tb = b if isinstance(b, tuple) else (b,)
    same = all(torch.equal(x.view(torch.uint8) if x.dtype != torch.uint8 else x, y.view(torch.uint8) if y.dtype != torch.uint8 else y)
               for x, y in zip(ta, tb))
    return a, same


def check_batch(b, stats, fails, tag):
    """Every entry point on one ray batch: fp16 and fp32 forward, inference and backward, and (fp16) the fused tail at reg_scale 1, 2."""
    from jnerf_b200 import ops
    cas, mean = b["cascades"], b["mean"]
    coords, ns_in, ns_c, bg, target = (_cu(b[k]) for k in ("coords", "ns_in", "ns_c", "bg", "target"))
    mean_t = torch.tensor([mean], dtype=torch.float32, device="cuda")
    R = b["ns_c"].shape[0]
    if R == 0:
        return
    for dt in (np.float16, np.float32):
        net_np = b["net"].astype(dt)
        net = _cu(net_np)
        cov = covered(b["ns_c"], net_np.shape[0])
        t = f"{tag}/{np.dtype(dt).name}"
        # forward
        rgb, same = _twice(lambda: ops.composite_fwd(net, coords, ns_in, ns_c, bg, cas))
        if not same:
            fails.append(f"{t}: two ngp_composite_fwd runs differ")
        rgb_np = _np(rgb)
        ex = ol.composite_f64(net_np, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas)
        check_rays(rgb_np, ex["rgb"], ex["rgb_err"], stats, "forward colour", t, fails)
        # inference
        (rgbi, alpha), same = _twice(lambda: ops.composite_infer(net, coords, ns_c, cas))
        if not same:
            fails.append(f"{t}: two ngp_composite_infer runs differ")
        exi = ol.composite_f64(net_np, b["coords"], None, b["ns_c"], None, cas)
        check_rays(_np(rgbi), exi["rgb"], exi["rgb_err"], stats, "inference colour", t, fails)
        check_rays(_np(alpha)[:, 0], exi["alpha"], exi["alpha_err"], stats, "alpha", t, fails)
        # backward on the kernel's own colour
        lg, _ = huber_f32(rgb_np, b["target"])
        rr_list = [rgb_np] + ([rgb_np + np.float32(b["rr_offset"])] if "rr_offset" in b else [])
        for rr in rr_list:
            dnet, same = _twice(lambda: ops.composite_bwd(net, coords, ns_c, _cu(lg), _cu(rr), mean_t, cas))
            if not same:
                fails.append(f"{t}: two ngp_composite_bwd runs differ")
            d = _np(dnet)
            if (d[~cov] != 0).any():
                fails.append(f"{t}: ngp_composite_bwd wrote {int((d[~cov] != 0).any(1).sum())} rows no ray covers")
            exb = ol.composite_f64(net_np, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas, l1=l1_of(mean), loss_grad=lg, rgb_ray=rr)
            check_dnet(d, exb, cov, stats, t + "/bwd", fails)
        if dt != np.float16:
            continue
        # the fused training tail
        for rs in (1.0, 2.0):
            def fused():
                dn = torch.full(net.shape, float(SENTINEL), dtype=torch.float16, device="cuda")
                return ops.composite_loss_bwd(net, coords, ns_in, ns_c, bg, target, mean_t, delta=DELTA, cascades=cas, dnet=dn, reg_scale=rs)
            (rgb2, loss, dnet2), same = _twice(fused)
            tt = f"{t}/fused rs={rs:g}"
            if not same:
                fails.append(f"{tt}: two ngp_composite_loss_bwd runs differ")
            rgb2_np, d2 = _np(rgb2), _np(dnet2)
            check_rays(rgb2_np, ex["rgb"], ex["rgb_err"], stats, "forward colour", tt, fails)
            lv, le = loss_bound(rgb2_np, b["target"])
            check_rays(_np(loss), lv, le, stats, "loss", tt, fails)
            if (d2[~cov].view(np.uint16) != SENTINEL.view(np.uint16)).any():
                fails.append(f"{tt}: ngp_composite_loss_bwd wrote rows no ray covers")
            lg2, _ = huber_f32(rgb2_np, b["target"])
            exf = ol.composite_f64(net_np, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas, l1=l1_of(mean, rs), loss_grad=lg2, rgb_ray=rgb2_np)
            check_dnet(d2, exf, cov, stats, tt, fails)
            if rs == 1.0:
                if not np.array_equal(rgb2_np.view(np.uint32), rgb_np.view(np.uint32)):
                    fails.append(f"{tt}: fused rgb differs from ngp_composite_fwd")
                d_pair = _np(ops.composite_bwd(net, coords, ns_c, _cu(lg2), rgb2, mean_t, cas))
                if not np.array_equal(d2[cov].view(np.uint16), d_pair[cov].view(np.uint16)):
                    fails.append(f"{tt}: fused dnet differs from ngp_composite_bwd on {int((d2[cov] != d_pair[cov]).any(1).sum())} rows")


def _report(case, stats, extra=""):
    print(f"[composite-fp64] {case}{extra}: " + "; ".join(f"{k} {v:.3g}" for k, v in stats.items()))


# ------------------------------------------------------------------------------------------------ training batches from the march
# id -> (rays, aabb, const_dt, cascades, scene, compaction aliased)
MARCH_CASES = {
    "lego": (4096, (0.0, 1.0), True, 5, "shell", True),
    "lego-solid": (4096, (0.0, 1.0), True, 5, "solid", True),
    "fox": (8192, (-1.5, 2.5), False, 5, "solid", True),
    "llff-7": (4096, None, False, 7, "llff", True),
    "adapted-13003": (13003, (0.0, 1.0), True, 5, "shell", True),
    "short-65005": (65005, (0.0, 1.0), True, 5, "small", True),
    "lego-copy": (4096, (0.0, 1.0), True, 5, "shell", False),
}


@functools.lru_cache(maxsize=None)
def _scene(kind, cascades):
    if kind == "llff":
        return shells_bitfield(cascades)[0]
    return {"shell": lambda: ol.sphere_bitfield(0.3, shell=0.03)[0], "solid": lambda: ol.sphere_bitfield(0.3)[0],
            "small": lambda: ol.sphere_bitfield(0.08)[0]}[kind]()


@functools.lru_cache(maxsize=None)
def march_case(case):
    """GPU march + compaction of one training-size batch, compared with the oracle; returns (bookkeeping mismatches, composite batch)."""
    from jnerf_b200 import ops
    R, aabb, const_dt, cas, scene, alias = MARCH_CASES[case]
    seed = sum(map(ord, case))
    if scene == "llff":
        half = 2.0 ** (cas - 1) / 2
        aabb = (0.5 - half, 0.5 + half)
        o, d = wide_rays(R, cas, seed=seed)
    else:
        o, d = ol.random_rays(R, seed=seed)
    bits = _scene(scene, cas)
    rng = ol.pcg32_seed(seed)
    coords, ridx, ns, cnt = ops.march(_cu(o), _cu(d), _cu(bits), aabb, MAX_SAMPLES, 0.00390625, 0.2, cas, const_dt, rng)
    cc, ns_c, cnt_c = ops.compact(coords, ns, CAP, alias=alias)
    torch.cuda.synchronize()
    assert ops.lib.load().ngp_debug_timeout_flag() == 0
    ref = ol.march(o, d, bits, aabb=aabb, max_samples=MAX_SAMPLES, cascades=cas, const_dt=const_dt, rng=rng)
    S = int(ref[3][1])
    bad = []
    if not np.array_equal(_np(cnt).view(np.uint32), ref[3]):
        bad.append(f"march counters {_np(cnt).view(np.uint32)} != {ref[3]}")
    if not np.array_equal(_np(ns).view(np.uint32), ref[2]):
        bad.append("march numsteps")
    if not np.array_equal(_np(ridx).view(np.uint32), ref[1]):
        bad.append("march ray indices")
    if not np.array_equal(_np(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32)):
        bad.append("march coordinates")
    rc = ol.compact(ref[0], ref[2], CAP)
    if not np.array_equal(_np(ns_c).view(np.uint32), rc[1]):
        bad.append("compacted numsteps")
    if not np.array_equal(_np(cnt_c).view(np.uint32), rc[2]):
        bad.append(f"compaction counters {_np(cnt_c).view(np.uint32)} != {rc[2]}")
    if not alias and not np.array_equal(_np(cc[:CAP]).view(np.uint32), rc[0].view(np.uint32)):
        bad.append("compacted coordinates")
    n_in, n_c = ref[2][:, 0], rc[1][:, 0]
    info = dict(S=S, cut=int(((n_c > 0) & (n_c < n_in)).sum()), zeroed=int(((n_c == 0) & (n_in > 0)).sum()), per=-(-R // 1024))
    g = np.random.default_rng(seed)
    net = np.empty((CAP, 4), np.float32)
    net[:, :3] = g.normal(0, 2.5, (CAP, 3))
    net[:, 3] = g.normal(0.5, 2.0, CAP)
    batch = dict(net=net, coords=_np(cc[:CAP]), ns_in=_np(ns), ns_c=_np(ns_c), bg=g.random((R, 3), dtype=np.float32),
                 target=g.random((R, 3), dtype=np.float32), cascades=cas, mean=0.001)
    return bad, batch, info


@pytest.mark.parametrize("case", list(MARCH_CASES))
def test_march_and_compaction_bookkeeping_at_training_size(case):
    """numsteps, ray indices, counters, accepted coordinates and the compacted numsteps / counters equal the oracle's bit for bit at
    R > 1024 (each scan thread walks several rays), with the 2^18 compaction cap inside one thread's segment."""
    bad, b, info = march_case(case)
    assert info["per"] >= 4 and info["S"] > CAP and info["cut"] + info["zeroed"] > 0, info
    assert not bad, bad


def test_march_max_samples_cut_inside_a_scan_segment():
    """The march's own max_samples cut on the third ray of one scan thread's four: that ray and every later one overflow (numsteps 0,
    ray index left at 0) while the two before it in the same segment keep theirs."""
    from jnerf_b200 import ops
    R = 4096
    o, d = ol.random_rays(R, seed=77)
    bits = _scene("shell", 5)
    rng = ol.pcg32_seed(77)
    full = ol.march(o, d, bits, max_samples=MAX_SAMPLES, rng=rng)
    n = full[2][:, 0].astype(np.int64)
    per = -(-R // 1024)
    i0 = next(i for i in range(R // 2, R) if i % per == 2 and n[i] > 0)
    max_samples = int(full[2][i0, 1]) + int(n[i0]) - 1
    ref = ol.march(o, d, bits, max_samples=max_samples, rng=rng)
    coords, ridx, ns, cnt = ops.march(_cu(o), _cu(d), _cu(bits), (0.0, 1.0), max_samples, 0.00390625, 0.2, 5, True, rng)
    assert ref[2][i0, 0] == 0 and ref[2][i0 - 1, 0] == n[i0 - 1]
    assert np.array_equal(_np(cnt).view(np.uint32), ref[3])
    assert np.array_equal(_np(ns).view(np.uint32), ref[2])
    assert np.array_equal(_np(ridx).view(np.uint32), ref[1])
    S = int(ref[2][i0 - 1].sum())                                          # rows of the accepted rays
    assert np.array_equal(_np(coords[:S]).view(np.uint32), ref[0][:S].view(np.uint32))
    _, ns_c, cnt_c = ops.compact(coords, ns, min(CAP, S - 1000), alias=True)
    rc = ol.compact(ref[0], ref[2], min(CAP, S - 1000))
    assert np.array_equal(_np(ns_c).view(np.uint32), rc[1]) and np.array_equal(_np(cnt_c).view(np.uint32), rc[2])


# ------------------------------------------------------------------------------------------------ the composite
def targets_at_delta(rgb, delta=DELTA):
    """Targets with fl(|rgb - target|) == delta exactly where a float within 4 ulps of rgb +- delta gives it, else rgb + delta; and
    the mask of the exact ones.  For rgb in [0.25, 1) no target does (rgb - target is exact there and delta = 0.1f has a bit below
    their grid), so the colours of the batch that uses this are kept below 0.25."""
    d = np.float32(delta)
    t, exact = (rgb + d).astype(np.float32), np.zeros(rgb.shape, bool)
    for idx in np.ndindex(rgb.shape):
        r = rgb[idx]
        for t0 in (np.float32(r + d), np.float32(r - d)):
            cands, up, dn = [t0], t0, t0
            for _ in range(4):
                up, dn = np.nextafter(up, np.float32(9)), np.nextafter(dn, np.float32(-9))
                cands += [up, dn]
            hit = [c for c in cands if np.abs(np.float32(r - c)) == d]
            if hit:
                t[idx], exact[idx] = hit[0], True
                break
    return t, exact


def _huber_edge_batches():
    """density_grid_mean exactly 0.01f (no l1) and the float below it (l1 on), and targets at |rgb - target| == delta exactly (the
    kernels are deterministic: the second run reproduces the colour the targets were made from)."""
    from jnerf_b200 import ops
    b = lengths_batch(list(np.resize(EDGE_LENGTHS[1:10], 45)), seed=400, adversarial=True)
    g = np.random.default_rng(401)
    b["net"][:, :3] = g.normal(-2.6, 0.3, (b["net"].shape[0], 3))          # colours ~ 0.07 and a dark background: rgb < 0.25
    b["bg"] = (g.random(b["bg"].shape) * 0.1).astype(np.float32)
    rgb = _np(ops.composite_fwd(_cu(b["net"].astype(np.float16)), _cu(b["coords"]), _cu(b["ns_in"]), _cu(b["ns_c"]), _cu(b["bg"]), 5))
    t, exact = targets_at_delta(rgb)
    t[::3, 2] = np.nextafter(t[::3, 2], np.float32(2))                    # and some a float off the edge
    assert exact.mean() > 0.25, exact.mean()
    return [dict(b, target=t, mean=float(mean)) for mean in (np.float32(0.01), np.nextafter(np.float32(0.01), np.float32(0)))]


def _trained_batch():
    """One training step of a lego runner after 100 steps: the fused tail's inputs exactly as Runner._net_pass passes them."""
    from jnerf_b200 import ops
    from test_gpu_parity_e2e import _trained_runner
    r = _trained_runner("lego", 100)
    seen = {}
    orig = ops.composite_loss_bwd

    def spy(net, coords, numsteps_in, numsteps_c, bg, target, mean, delta=0.1, cascades=5, **kw):
        seen.update(net=net.clone(), coords=coords.clone(), ns_in=numsteps_in.clone(), ns_c=numsteps_c.clone(), bg=bg.clone(),
                    target=target.clone(), mean=mean.clone(), delta=delta, cascades=cascades, reg_scale=kw.get("reg_scale", 1.0))
        return orig(net, coords, numsteps_in, numsteps_c, bg, target, mean, delta=delta, cascades=cascades, **kw)
    ops.composite_loss_bwd = spy
    try:
        r.train_step()
        torch.cuda.synchronize()
    finally:
        ops.composite_loss_bwd = orig
    assert seen["delta"] == DELTA and seen["reg_scale"] == 1.0 and seen["net"].dtype == torch.float16
    return dict(net=_np(seen["net"]).astype(np.float32), coords=_np(seen["coords"]), ns_in=_np(seen["ns_in"]), ns_c=_np(seen["ns_c"]),
                bg=_np(seen["bg"]), target=_np(seen["target"]), cascades=int(seen["cascades"]), mean=float(_np(seen["mean"])[0]))


COMPOSITE_CASES = list(MARCH_CASES) + ["edge-lengths", "adversarial", "huber-mean-edges", "trained-lego"]


@pytest.mark.parametrize("case", COMPOSITE_CASES)
def test_composite_against_fp64(case):
    if case in MARCH_CASES:
        batches, extra = [march_case(case)[1]], " ({S} raw rows, {cut} rays cut short, {zeroed} cut to zero)".format(**march_case(case)[2])
    elif case == "edge-lengths":
        batches, extra = edge_batches(), ""
    elif case == "adversarial":
        batches, extra = [adversarial_batch()], ""
    elif case == "huber-mean-edges":
        batches, extra = _huber_edge_batches(), ""
    else:
        batches = [_trained_batch()]
        extra = f" (R = {batches[0]['ns_c'].shape[0]}, mean {batches[0]['mean']:.4g})"
    stats, fails = {}, []
    for k, b in enumerate(batches):
        check_batch(b, stats, fails, f"{case}#{k}")
    _report(case, stats, extra)
    assert not fails, fails[:10]
