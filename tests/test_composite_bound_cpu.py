"""Rehearsal of the composite error bound of test_gpu_composite_reference.py on the CPU: the oracle's serial fp32 composite
(orc_composite_fwd / _infer / _bwd, libm expf and IEEE division, one fmaf per sample) is another fp32 evaluation of the same
expressions in another association order, so every one of its colours, alphas, losses and dL/dnet entries must lie within the
bound too.  This is the check that neither the float64 reference nor the bound is too tight.  It also checks the float64 composite
against a plain numpy restatement."""
import numpy as np
import pytest

import oracle_lib as ol
from test_gpu_composite_reference import (EDGE_LENGTHS, SAFETY, adversarial_batch, check16, check_dnet, check_rays, covered, edge_batches,
                                          huber_f32, l1_of, lengths_batch, loss_bound)


def _oracle_batch(b, dt, stats, fails, tag, reg_scale=1.0):
    net = b["net"].astype(dt)
    cas, mean = b["cascades"], b["mean"]
    t = f"{tag}/{np.dtype(dt).name}"
    rgb = ol.composite_fwd(net, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas)
    ex = ol.composite_f64(net, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas)
    check_rays(rgb, ex["rgb"], ex["rgb_err"], stats, "forward colour", t, fails)
    rgbi, alpha = ol.composite_infer(net, b["coords"], b["ns_c"], cas)
    exi = ol.composite_f64(net, b["coords"], None, b["ns_c"], None, cas)
    check_rays(rgbi, exi["rgb"], exi["rgb_err"], stats, "inference colour", t, fails)
    check_rays(alpha[:, 0], exi["alpha"], exi["alpha_err"], stats, "alpha", t, fails)
    g, l = ol.huber_grad(rgb, b["target"], 0.1)
    lg, _ = huber_f32(rgb, b["target"])
    assert np.array_equal(lg.ravel().view(np.uint32), g.view(np.uint32))            # the numpy fp32 Huber is the oracle's
    l = l.reshape(-1, 3)
    loss = (l[:, 0] + l[:, 1]) + l[:, 2]
    lv, le = loss_bound(rgb, b["target"])
    check_rays(loss, lv, le, stats, "loss", t, fails)
    cov = covered(b["ns_c"], net.shape[0])
    ol.oracle().orc_set_reg_scale(ol._f32(reg_scale))
    try:
        for rr in [rgb] + ([rgb + np.float32(b["rr_offset"])] if "rr_offset" in b else []):
            d = ol.composite_bwd(net, b["coords"], b["ns_c"], lg.reshape(-1, 3), rr, mean, cas)
            exb = ol.composite_f64(net, b["coords"], b["ns_in"], b["ns_c"], b["bg"], cas, l1=l1_of(mean, reg_scale), loss_grad=lg.reshape(-1, 3),
                                   rgb_ray=rr)
            check_dnet(d, exb, cov, stats, t + "/bwd", fails)
    finally:
        ol.oracle().orc_set_reg_scale(ol._f32(1.0))


def _batches(name):
    if name == "edge-lengths":
        return edge_batches()
    if name == "adversarial":
        return [adversarial_batch()]
    b = lengths_batch(list(np.random.default_rng(5).integers(0, 700, 203)), seed=5)
    return [b, dict(b, mean=float(np.float32(0.01))), dict(b, mean=float(np.nextafter(np.float32(0.01), np.float32(0))))]


@pytest.mark.parametrize("dt", [np.float16, np.float32])
@pytest.mark.parametrize("name", ["edge-lengths", "adversarial", "random-lengths"])
def test_bound_holds_for_the_serial_fp32_oracle(name, dt):
    stats, fails = {}, []
    for k, b in enumerate(_batches(name)):
        _oracle_batch(b, dt, stats, fails, f"{name}#{k}", reg_scale=2.0 if k == 1 else 1.0)
    print(f"[composite-bound-cpu] {name}/{np.dtype(dt).name}: " + "; ".join(f"{k} {v:.3g}" for k, v in sorted(stats.items())))
    assert not fails, fails[:10]
    assert stats[f"dnet colour {np.dtype(dt).name}"] > 0 and stats["forward colour"] > 0


def _numpy_composite(b, dt):
    """The composite restated in float64 numpy, ray by ray: colour (with the background rule) and dL/dnet for rr = that colour."""
    net = b["net"].astype(dt).astype(np.float64)
    mn = np.float32(1.73205080757) / np.float32(1024)                      # nerf_unwarp_dt at 5 cascades
    span = mn * np.float32(16) - mn
    R = b["ns_c"].shape[0]
    ls = np.float64(np.float32(128) / np.float32(R))
    lg = np.random.default_rng(1).standard_normal((R, 3)).astype(np.float32)
    rgb = np.zeros((R, 3))
    dnet = np.full((net.shape[0], 4), np.nan)
    for i in range(R):
        n, base = b["ns_c"][i]
        if n == 0:
            rgb[i] = b["bg"][i]
            continue
        rows = net[base:base + n]
        dt_ = (b["coords"][base:base + n, 3].astype(np.float64) * np.float64(span) + np.float64(mn)).astype(np.float32).astype(np.float64)
        c = 1 / (1 + np.exp(-rows[:, :3]))
        alpha = -np.expm1(-np.exp(rows[:, 3]) * dt_)
        T = np.concatenate([[1.0], np.cumprod(1 - alpha)])
        w = alpha * T[:-1]
        rgb[i] = (w[:, None] * c).sum(0) + (T[-1] * b["bg"][i] if n == b["ns_in"][i, 0] else 0)
        run = np.cumsum(w[:, None] * c, 0)
        suffix = rgb[i] - run
        dot = (lg[i] * (T[1:, None] * c - suffix)).sum(1)
        dnet[base:base + n, :3] = ls * w[:, None] * lg[i] * c * (1 - c)
        dnet[base:base + n, 3] = ls * np.exp(np.clip(rows[:, 3], -15, 15)) * dt_ * dot
    return rgb, lg, dnet


def test_f64_composite_matches_a_numpy_restatement():
    """orc_composite_f64's exact values against the formulae written out with numpy (no fp32 rounding anywhere but dt), on rays with a
    moderate density where both are accurate to far below the bound: a transposed index, a wrong background rule or a suffix taken
    before instead of after the sample would differ by orders of magnitude more."""
    b = lengths_batch(EDGE_LENGTHS[:14] * 2, seed=9, opaque=False)
    for dt in (np.float16, np.float32):
        rgb, lg, dnet = _numpy_composite(b, dt)
        net = b["net"].astype(dt)
        ex = ol.composite_f64(net, b["coords"], b["ns_in"], b["ns_c"], b["bg"], 5, loss_grad=lg, rgb_ray=rgb.astype(np.float32))
        assert np.abs(ex["rgb"] - rgb).max() <= 1e-12
        cov = covered(b["ns_c"], net.shape[0])
        # rr enters as fp32: the suffix differs by at most the rounding of rr
        rgb32 = rgb.astype(np.float32).astype(np.float64)
        assert np.all(np.isfinite(ex["dnet"][cov])) and np.all(np.isfinite(ex["dnet_err"][cov]))
        assert np.abs(ex["dnet"][cov, :3] - dnet[cov, :3]).max() <= 1e-12 * np.abs(dnet[cov, :3]).max()
        scale = np.abs(dnet[cov, 3]).max()
        assert np.abs(ex["dnet"][cov, 3] - dnet[cov, 3]).max() <= 1e-3 * scale, np.abs(ex["dnet"][cov, 3] - dnet[cov, 3]).max() / scale
        assert np.abs(rgb32 - rgb).max() < 1e-7
        assert (ex["dnet_err"][cov] > 0).all() and (ex["rgb_err"][b["ns_c"][:, 0] > 0] > 0).all()
        assert SAFETY * ex["rgb_err"].max() < 2e-4                        # gamma_1024 ~ 6e-5 of the colour: not a vacuous bound


def test_fp16_rounding_check():
    """check16 accepts exactly the correct roundings of the interval: subnormals with their 2^-24 spacing, +-inf above 65520, and a
    zero only where the interval reaches zero."""
    x = np.array([1e-6, 1e-6, 1e-6, 7e4, 65519.0, 3.0, 0.0])
    e = np.array([1e-12, 1e-12, 1e-6, 0.0, 0.0, 0.0, 0.0])
    g = np.array([np.float16(1e-6), np.float16(0), np.float16(0), np.float16(np.inf), np.float16(65504), np.float16(3), np.float16(0)])
    ok, _ = check16(g, x, e)
    assert ok.tolist() == [True, False, True, True, True, True, True]
