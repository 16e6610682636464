"""The float64 harness of tests/test_nerf_mlp_reference.py (tests/nerf_mlp_ref.py), checked without a GPU: the slab decoder against the
kernels' group constants, the one-rounding fp16 reference and the rounding-interval check at their edges, and the layer tables composed
into the whole network against the reference-named chain of plugin/nerf.py (forward, and backward against autograd)."""
import math
import os
import re

import numpy as np
import pytest
import torch

import nerf_mlp_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_constants():
    src = open(os.path.join(ROOT, "jnerf_b200", "csrc", "nerf_mlp.cuh")).read()
    return {k: int(v) for k, v in re.findall(r"\b([SD]_[A-Z0-9]+) = (\d+)", src)}


def test_column_map_is_the_kernels_group_layout():
    c = _header_constants()
    assert (c["S_GROUPS"], c["D_GROUPS"]) == (R.S_GROUPS, R.D_GROUPS)
    assert (8 * c["S_ENC"], 8 * c["S_F"], 8 * c["S_DIR"], 8 * c["S_V"]) == (R.ENC, R.F, R.DIR, R.V)
    assert all(8 * (c["S_H"] + 32 * l) == R.H(l) for l in range(8))
    assert all(8 * (c["D_H"] + 32 * l) == R.DY(l) for l in range(8))
    assert (8 * c["D_8"], 8 * c["D_9"], 8 * c["D_10"]) == (R.DY(8), R.DY(9), R.DY(10))


@pytest.mark.parametrize("groups", [R.S_GROUPS, R.D_GROUPS])
def test_decoder_on_a_hand_built_block(groups):
    """Block t, group g, slab row r, lane k holds the id of (row 128 t + r, column 8 g + k); one trailing block is not decoded."""
    tiles = 3
    t, g, r, k = np.meshgrid(np.arange(tiles + 1), np.arange(groups), np.arange(R.ROWS), np.arange(8), indexing="ij")
    ids = (R.ROWS * t + r) * (8 * groups) + 8 * g + k
    out = R.decode(torch.from_numpy(ids.astype(np.int64).ravel()), groups, tiles)
    assert out.shape == (tiles * R.ROWS, 8 * groups)
    want = np.arange(tiles * R.ROWS)[:, None] * (8 * groups) + np.arange(8 * groups)[None, :]
    assert np.array_equal(out.numpy(), want)
    # a uint8 buffer is read as fp16: group 300, row 5, lane 2 of tile 1 is column 2402 of row 133
    h = torch.zeros(2 * groups * R.ROWS * 8, dtype=torch.float16)
    h[((1 * groups + 300) * R.ROWS + 5) * 8 + 2] = 3.5
    d = R.decode(h.view(torch.uint8), groups, 2)
    assert d[133, 2402] == 3.5 and float(d.abs().sum()) == 3.5


def test_rn16_is_one_rounding():
    ties = [1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(2 + 2.0 ** -10), 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -14 + 2.0 ** -25, 65520.0, 65519.99]
    for y, want in zip(ties, [1.0, 1 + 2.0 ** -9, -2.0, 0.0, 2.0 ** -23, 2.0 ** -14, math.inf, 65504.0]):
        assert float(R.rn16(torch.tensor([y], dtype=torch.float64))) == want, y
    # just above a tie: the direct rounding goes up, fp32 first lands on the tie and goes to even
    y = 1 + 2.0 ** -11 + 2.0 ** -40
    assert float(R.rn16(torch.tensor([y], dtype=torch.float64))) == 1 + 2.0 ** -10
    assert float(np.float16(np.float32(y))) == 1.0
    rng = np.random.default_rng(0)
    ys = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.uniform(-9, 5, 20000),          # subnormal to overflow
                         rng.integers(-2 ** 12, 2 ** 12, 5000) * 2.0 ** -25,                       # subnormal ties and halfway points
                         (rng.integers(2 ** 10, 2 ** 11, 5000) + 0.5) * 2.0 ** rng.integers(-24, 5, 5000), [0.0, -0.0]])
    got = R.rn16(torch.from_numpy(ys)).numpy()
    want = R.numpy_rn16(ys)
    assert np.array_equal(got, want)
    assert np.array_equal(np.signbit(got), np.signbit(want))


def test_rounding_interval_check():
    t = lambda *v: torch.tensor(v, dtype=torch.float64)
    h = lambda *v: torch.tensor(v, dtype=torch.float16)
    ok, ratio = R.check_rounding(h(1.0, 1.0, 1.0 + 2 ** -10), t(1.0004, 1.001, 1.0004), t(0.0, 0.0, 0.0))
    assert ok.tolist() == [True, False, False]                       # 1.0004 rounds to 1; 1.001 to 1 + 2^-10
    assert ratio[0] == 0 and math.isinf(ratio[1])
    ok, ratio = R.check_rounding(h(1.0 + 2 ** -10), t(1.0004), t(0.0002))   # 1.0004 + 0.0002 lies past the halfway point 1 + 2^-11
    assert bool(ok) and float(ratio) < 1
    ok, ratio = R.check_rounding(h(1.0 + 2 ** -10), t(1.0004), t(0.00005))
    assert not bool(ok) and float(ratio) > 1
    # exact ties go to even on both ends
    ok, _ = R.check_rounding(h(1.0, 1.0 + 2 ** -10), t(1 + 2.0 ** -11, 1 + 2.0 ** -11), t(0.0, 0.0))
    assert ok.tolist() == [True, False]
    # fp16 subnormals: 2^-24 is the only value within 2^-26 of 1.1 * 2^-24
    ok, _ = R.check_rounding(h(0.0, 2 ** -24, 2 ** -23), t(1.1 * 2 ** -24, 1.1 * 2 ** -24, 1.1 * 2 ** -24), t(2.0 ** -26, 2.0 ** -26, 2.0 ** -26))
    assert ok.tolist() == [False, True, False]
    # ReLU: a negative interval allows only zero, of either sign; one reaching past zero allows its positive roundings too
    ok, ratio = R.check_rounding(h(0.0, -0.0, 2 ** -24, -(2 ** -24)), t(-0.3, -0.3, -0.3, -0.3), t(0.1, 0.1, 0.1, 0.1), relu=True)
    assert ok.tolist() == [True, True, False, False] and ratio[0] == 0
    ok, _ = R.check_rounding(h(0.0, 0.001), t(-0.0005, -0.0005), t(0.0016, 0.0016), relu=True)
    assert ok.tolist() == [True, True]
    # +-0 without a ReLU, and a NaN never passes
    ok, _ = R.check_rounding(h(0.0, -0.0, math.nan), t(-0.0, 0.0, 0.0), t(0.0, 0.0, 1.0))
    assert ok.tolist() == [True, True, False]


def test_pad_mask_is_what_pack_leaves_zero():
    from jnerf_b200.plugin import nerf
    ones = {name: (torch.ones(shape), torch.ones(shape[0])) for name, (shape, _, _, _) in nerf.REF_LAYERS.items()}
    assert torch.equal(R.pad_mask(), nerf.pack(ones) == 0)
    assert int(R.pad_mask().sum()) == 15 * 257 + 13 * 129 + 2 * 256 + 5 * 128


def _random_model(seed=0):
    from jnerf_b200.plugin import nerf
    g = torch.Generator().manual_seed(seed)
    ref = {}
    for name, ((o, i), _, _, _) in nerf.REF_LAYERS.items():
        ref[name] = ((torch.rand((o, i), generator=g) * 2 - 1) * math.sqrt(3 / i) * 1.5, (torch.rand(o, generator=g) * 2 - 1) * 0.3)
    P = nerf.pack(ref)
    return nerf, {k: (W.double().requires_grad_(), b.double().requires_grad_()) for k, (W, b) in nerf.unpack(P).items()}, P


def test_layer_tables_compose_to_the_reference_network():
    """FWD / DGRAD / wgrad_flat composed over the flat vector against plugin/nerf.py's named chain (float64 on both sides, so a
    misplaced column or weight row, not rounding, is what would differ)."""
    nerf, ref, P = _random_model()
    g = torch.Generator().manual_seed(1)
    n = 300
    enc = torch.zeros((n, 64), dtype=torch.float64)
    enc[:, :63] = torch.rand((n, 63), generator=g, dtype=torch.float64) * 2 - 1
    encd = torch.zeros((n, 32), dtype=torch.float64)
    encd[:, :27] = torch.rand((n, 27), generator=g, dtype=torch.float64) * 2 - 1
    dout = torch.randn((n, 4), generator=g, dtype=torch.float64)
    lin = lambda name, x: x @ ref[name][0].t() + ref[name][1]
    h = enc[:, :63]
    for i in range(8):
        h = torch.relu(lin(f"pts_linears.{i}", h))
        if i == 4:
            h = torch.cat([enc[:, :63], h], -1)
    alpha = lin("alpha_linear", h)
    v = torch.relu(lin("views_linears.0", torch.cat([lin("feature_linear", h), encd[:, :27]], -1)))
    want = torch.cat([lin("rgb_linear", v), alpha], -1)
    (want * dout).sum().backward()

    sv, out = R.forward_chain(P, enc, encd)
    assert torch.allclose(out, want.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(sv[:, R.V:R.V + 128], v.detach(), rtol=1e-12, atol=1e-12)
    dys = R.backward_chain(P, sv, dout)
    grad, mag, _ = R.wgrad_flat(dys, sv)
    pad = R.pad_mask()
    assert torch.equal(grad[pad], torch.zeros_like(grad[pad])) and bool((mag[~pad] > 0).any())
    got = nerf.unpack(grad)
    for name, (W, b) in ref.items():
        assert torch.allclose(got[name][0].double(), W.grad, rtol=1e-6, atol=1e-9), name
        assert torch.allclose(got[name][1].double(), b.grad, rtol=1e-6, atol=1e-9), name
    # the chain's own pad columns stay zero
    assert not dys[:, R.DY(8) + 1:R.DY(8) + 16].any() and not dys[:, R.DY(8) + 272:R.DY(9)].any() and not dys[:, R.DY(10) + 3:].any()


def test_freq_encoding_matches_plugin_encoder():
    from jnerf_b200.plugin import nerf
    x = torch.rand((50, 3), generator=torch.Generator().manual_seed(2))
    y, e = R.freq_encoding(x, 10)
    assert y.shape == (50, 64) and not y[:, 63].any() and not e[:, 63].any() and not e[:, :3].any()
    assert torch.allclose(y[:, :63].float(), nerf.freq_encode(x, 10), atol=2e-6)
    assert bool((e[:, 3:63] > 0).all()) and float((e / y.abs().clamp_min(1e-30))[:, 3:63].max()) <= 2 * 2.0 ** -23
