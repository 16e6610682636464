"""The vanilla NeRF network kernels (csrc/nerf_mlp.cu, nerf_mlp.cuh; mip_mlp.cu as Mip-NeRF's encode stage) against float64, layer by
layer, at the training batch sizes of both models that use them, with a bound on every entry.

The forward saves every layer's input and the backward's scratch keeps every layer's pre-activation gradient (tests/nerf_mlp_ref.py
decodes both).  Every check starts from the kernel's own fp16 operands, so it is exact and independent of the order of summation:
- forward, per layer: the saved output is a correct fp16 rounding of a value within (K + 2) 2^-23 (sum |x w| + |b| + F) of the exact
  x W^T + b, after the ReLU where there is one; the encodings within 2 fp32 ulps of float64 sin / cos of the fp32 argument (Mip-NeRF's
  integrated encoding within the 2e-4 that test_mip_gpu.py allows the fp32 encoder), their padding exactly zero;
- dgrad, per layer: the same from the kernel's dY of the layer above, exactly zero where the saved activation is not positive; the
  output gradient enters exactly; rows at or past the row count are exactly zero;
- wgrad: every entry of every chunk's partial sum part[c] against the float64 sum over exactly that chunk's tiles, and the reduced
  gradient against the whole sum, within (L + NCHUNK + 2) 2^-23 (sum |dY x| + F), L the chunk's number of rows with a nonzero gradient
  and F the tensor core's alignment floor (tests/nerf_mlp_ref.py); the padding of the flat vector exactly zero.  At 2^18 rows L is
  32 768 and the bound a loose 2^-8; so every case runs a second backward whose output gradient is zero except on one row per tile
  (at in-tile position t mod 128), every row of the last tile and a few random rows.  Then L is a few hundred and the bound about
  2^-14 of sum |dY x|: a lost or misplaced tile misses it by orders of magnitude.

Two weight sets: the reference initialisation, and the same weights doubled with every bias lowered by 0.4, which leaves most ReLUs of
every layer dead and lets live activations reach O(10).

The accumulation bound first assumed only an fp32 accumulator that may truncate at every step, (K + 2) 2^-23 sum |x w|.  On an H100
that held everywhere but in the Mip-NeRF probe: one weight-gradient entry per weight set, a sum of two products of about 4e-8 from
fp16-subnormal output gradients, came back with 16 significant bits, 1.6 and 1.3 times that bound.  The kernel sums the right terms;
the tensor core aligns a k-block's products no lower than a product with a zero fp16 operand, so the bound now carries the floor F of
tests/nerf_mlp_ref.py.  Worst error / bound over all cases on an H100 (80 GB HBM3, 700 W power limit), the error of an fp16 result
being the distance from the exact value to the nearest real that rounds to it: forward 0.014, encoding 0.60, dgrad 0.047, dense
wgrad 0.034, probe wgrad 0.18.  The file takes about 16 s there."""
import math

import numpy as np
import pytest
import torch

import nerf_mlp_ref as R

pytestmark = pytest.mark.gpu

BLOCK = 1 << 15                    # rows per float64 block
SENTINEL = 0x7E01                  # a NaN payload no kernel result carries: rows past the row count of `out` must keep it
MIP_R, MIP_S = 288, 128            # mip_cfg: 288 rays x 128 samples, two levels

# id -> (rows launched, device row count or None)
CASES = {
    "n1": (1, None), "n127": (127, None), "n128": (128, None), "n129": (129, None),
    "n896": (896, None),                         # 7 tiles: fewer tiles than chunks, some chunks empty
    "n4813": (128 * 37 + 77, None),
    "dev0": (1000, 0), "dev333": (1000, 333), "dev-over": (1000, 5000),
    "train-2^18": (1 << 18, None),               # nerf_cfg's target_batch_size: 2048 tiles, 256 per chunk
    "mip": (2 * MIP_R * MIP_S, None),           # both levels of one Mip-NeRF step through one backward
}


def _tiles(n):
    return -(-n // R.ROWS)


def _nchunk(n_max):
    from jnerf_b200 import ops
    rest = ops.nerf_workspace_bytes(n_max)[1] - _tiles(n_max) * R.D_GROUPS * R.GB
    assert rest > 0 and rest % (R.N_PARAMS * 4) == 0
    return rest // (R.N_PARAMS * 4)


def _weights(kind, mip=False):
    from jnerf_b200.plugin import mip as mipm
    from jnerf_b200.plugin import nerf
    gen = torch.Generator(device="cuda").manual_seed(11)
    ref = nerf.init_reference_params(gen, mipm.REF_LAYERS, mipm.REF_ORDER) if mip else nerf.init_reference_params(gen)
    if kind == "dead":
        ref = {k: (2 * W, b - 0.4) for k, (W, b) in ref.items()}
    return (mipm.pack if mip else nerf.pack)(ref)


def _coords(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.zeros((n, 7), device="cuda")
    c[:, :3] = torch.rand((n, 3), device="cuda", generator=g) * 4 - 2
    c[:, 4:] = torch.nn.functional.normalize(torch.randn((n, 3), device="cuda", generator=g), dim=-1)
    return c


def _probe(dout, n, seed):
    """dout zero except on row 128 t + t mod 128 of every tile t, every row of the last tile and 16 random rows"""
    T = _tiles(n)
    keep = torch.zeros(dout.shape[0], dtype=torch.bool, device="cuda")
    t = torch.arange(T, device="cuda")
    rows = t * R.ROWS + t % R.ROWS
    keep[rows[rows < n]] = True
    keep[(T - 1) * R.ROWS:n] = True
    keep[torch.randint(0, n, (16,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))] = True
    return torch.where(keep[:, None], dout, torch.zeros_like(dout))


def _run(case, kind):
    """Forward with saved activations, then a dense and a probe backward into caller-owned scratch."""
    from jnerf_b200 import ops
    n_max, n_dev = CASES[case]
    n = n_max if n_dev is None else min(n_dev, n_max)
    P = _weights(kind, mip=case == "mip")
    out = torch.full((n_max, 4), 0.0, dtype=torch.float16, device="cuda")
    out.view(torch.int16).fill_(SENTINEL)
    dev = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(n_max + (n_dev or 0))
    if case == "mip":
        enc = _mip_forward(P, out)
        saved = enc.pop("saved")
        dout = enc.pop("dout")
    else:
        c = _coords(n_max, seed=n_max)
        _, saved = ops.nerf_fwd(c, P, n_dev=dev, save=True, out=out)
        enc = dict(pos=lambda r0, r1: R.freq_encoding(_live(c, n, r0, r1)[:, :3], 10),
                   dir=lambda r0, r1: R.freq_encoding(_live(c, n, r0, r1)[:, 4:7], 4))
        dout = (torch.randn((n_max, 4), device="cuda", generator=g) * 0.1).half()
    runs = {}
    for name, d in (("dense", dout), ("probe", _probe(dout, max(n, 1), n_max))):
        scratch = torch.empty(ops.nerf_workspace_bytes(n_max)[1], dtype=torch.uint8, device="cuda")
        grad = ops.nerf_bwd(P, saved, d, n_dev=dev, scratch=scratch)
        runs[name] = (d, scratch, grad)
    torch.cuda.synchronize()
    return dict(n=n, n_max=n_max, P=P, out=out, saved=saved, enc=enc, runs=runs)


def _live(c, n, r0, r1):
    """coordinate rows [r0, r1) as the kernel encodes them: rows at or past n are zero"""
    x = torch.zeros((r1 - r0, 7), dtype=c.dtype, device=c.device)
    x[:max(0, min(n, r1) - r0)] = c[r0:min(n, r1)]
    return x


def _mip_forward(P, out):
    """MipRunner.train_step's network part: both levels' forwards into the halves of one saved buffer, the loss gradient of both
    levels with grad_scale = R."""
    import mip_cpu_backend as ref
    from test_mip_gpu import _rays
    from jnerf_b200 import ops
    rays = _rays(MIP_R, seed=3)
    rng = ops.pcg32_seed(9)
    n = MIP_R * MIP_S
    half = ops.nerf_workspace_bytes(n)[0]
    saved = torch.empty(2 * half, dtype=torch.uint8, device="cuda")
    t_c = ops.mip_sample(rays, MIP_S, False, True, rng)
    ops.mip_fwd(rays, t_c, P, out=out[:n], saved=saved[:half])
    w = ops.mip_composite_fwd(out[:n], t_c, rays, 0.001, -1.0, False)[3]
    t_f = ops.mip_resample(t_c, w, 0.01, True, rng)
    ops.mip_fwd(rays, t_f, P, out=out[n:], saved=saved[half:])
    target = torch.rand((MIP_R, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    _, _, dout = ops.mip_composite_loss_bwd(out, torch.cat([t_c, t_f]), rays, target, None, 0.001, -1.0, False, 0.1, grad_scale=float(MIP_R))
    ipe = torch.zeros((2 * n, 64), dtype=torch.float64, device="cuda")
    for k, t in enumerate((t_c, t_f)):
        ipe[k * n:(k + 1) * n, :48] = ref.encode(rays.double(), t.double(), "cone", True, 0, 8)[0]
    ipe_e = torch.zeros_like(ipe)
    ipe_e[:, :48] = 2e-4
    view = rays[:, 6:9].repeat_interleave(MIP_S, 0).repeat(2, 1)
    return dict(pos=lambda r0, r1: (ipe[r0:r1], ipe_e[r0:r1]), dir=lambda r0, r1: R.freq_encoding(view[r0:r1], 4), saved=saved,
                dout=dout.contiguous())


class Tally:
    def __init__(self):
        self.worst, self.fails = {}, []

    def add(self, family, what, ok, ratio):
        if ratio.numel():
            self.worst[family] = max(self.worst.get(family, 0.0), float(ratio.max()))
        bad = int((~ok).sum())
        if bad:
            self.fails.append(f"{what}: {bad} of {ok.numel()} entries outside the bound")

    def exact(self, what, ok):
        if not bool(ok.all()):
            self.fails.append(f"{what}: {int((~ok).sum())} entries differ")


def _bits(t):
    return t.contiguous().view(torch.int16)


def _check_forward(r, tally):
    n, P, T = r["n"], r["P"], _tiles(r["n"])
    sv = R.decode(r["saved"], R.S_GROUPS, T)
    dead = torch.zeros(8, dtype=torch.float64, device="cuda")
    for r0 in range(0, T * R.ROWS, BLOCK):
        r1 = min(r0 + BLOCK, T * R.ROWS)
        s = sv[r0:r1]
        for name, c, w in (("pos", R.ENC, 64), ("dir", R.DIR, 32)):
            y, e = r["enc"][name](r0, r1)
            tally.add("encoding", f"enc_{name}", *R.check_rounding(s[:, c:c + w], y, e))
            pad = (e == 0) & (y == 0)
            tally.exact(f"enc_{name} padding", _bits(s[:, c:c + w])[pad] == 0)
        for l in range(11):
            W, b = R.layer_params(P, l)
            x = R.layer_input(s, l)
            for w0, nr, (dst, c), relu in R.FWD[l]:
                y, e = R.fwd_layer(x, W[w0:w0 + nr], b[w0:w0 + nr])
                if dst == "saved":
                    tally.add("forward", f"layer {l} rows {w0}+{nr}", *R.check_rounding(s[:, c:c + nr], y, e, relu))
                else:                                                  # out holds rows < n only
                    m = max(0, min(n, r1) - r0)
                    tally.add("forward", f"layer {l} -> out[:, {c}:{c + nr}]", *R.check_rounding(r["out"][r0:r0 + m, c:c + nr], y[:m], e[:m]))
        live = min(n, r1) - r0
        for l in range(8):
            dead[l] += (s[:live, R.H(l):R.H(l) + 256] <= 0).double().sum()
    tally.exact("out rows past the row count", _bits(r["out"][n:]) == SENTINEL)
    return (dead / max(n, 1) / 256).tolist(), sv


def _check_backward(r, run, sv, tally, fam):
    n, n_max, P, T = r["n"], r["n_max"], r["P"], _tiles(r["n"])
    dout, scratch, grad = r["runs"][run]
    nchunk = _nchunk(n_max)
    dys_bytes = _tiles(n_max) * R.D_GROUPS * R.GB
    part = scratch[dys_bytes:dys_bytes + nchunk * R.N_PARAMS * 4].view(torch.float32).view(nchunk, R.N_PARAMS)
    dys = R.decode(scratch[:dys_bytes], R.D_GROUPS, T)
    nz = (dout[:n] != 0).any(1)
    # dgrad, per layer from the kernel's own dY of the layer above
    for r0 in range(0, T * R.ROWS, BLOCK):
        r1 = min(r0 + BLOCK, T * R.ROWS)
        d, s, m = dys[r0:r1], sv[r0:r1], max(0, min(n, r1) - r0)
        head = torch.zeros((r1 - r0, R.DYS_COLS - R.DY(10)), dtype=torch.float16, device="cuda")
        head[:m, :3] = dout[r0:r0 + m, :3]
        tally.exact(f"{run} dY10 = [drgb, 0]", _bits(d[:, R.DY(10):]) == _bits(head))
        a8 = torch.zeros((r1 - r0, 16), dtype=torch.float16, device="cuda")
        a8[:m, 0] = dout[r0:r0 + m, 3]
        tally.exact(f"{run} layer-8 dY = [dalpha, 0 x 15, ..]", _bits(d[:, R.DY(8):R.DY(8) + 16]) == _bits(a8))
        tally.exact(f"{run} layer-8 dY tail", _bits(d[:, R.DY(8) + 272:R.DY(9)]) == 0)
        for l, c0, nc, mask, dst in R.DGRAD:
            W = R.layer_params(P, l)[0]
            y, e = R.dgrad_layer(d[:, R.DY(l):R.DY(l) + R.OUT[l]], W[:, c0:c0 + nc])
            got = d[:, dst:dst + nc]
            ok, ratio = R.check_rounding(got, y, e)
            if mask is not None:
                live = s[:, mask:mask + nc] > 0
                tally.exact(f"{run} layer {l} dgrad under dead ReLUs", _bits(got)[~live] == 0)
                ok, ratio = ok | ~live, torch.where(live, ratio, torch.zeros_like(ratio))
            tally.add("dgrad", f"{run} layer {l} dgrad", ok, ratio)
        tally.exact(f"{run} dys rows past the row count", _bits(d[m:]) == 0)
    # wgrad: every chunk's partial sums over exactly its tiles, then the reduction
    g_all = torch.zeros(R.N_PARAMS, dtype=torch.float64, device="cuda")
    a_all, f_all = torch.zeros_like(g_all), torch.zeros_like(g_all)
    L_max = 0
    for c in range(nchunk):
        t0, t1 = c * T // nchunk, (c + 1) * T // nchunk
        g_c, a_c, f_c = torch.zeros_like(g_all), torch.zeros_like(g_all), torch.zeros_like(g_all)
        for r0 in range(t0 * R.ROWS, t1 * R.ROWS, BLOCK):
            r1 = min(r0 + BLOCK, t1 * R.ROWS)
            g, a, f = R.wgrad_flat(dys[r0:r1], sv[r0:r1])
            g_c += g
            a_c += a
            f_c = torch.maximum(f_c, f)
        L = int(nz[t0 * R.ROWS:t1 * R.ROWS].sum())
        L_max = max(L_max, L)
        _wgrad_entries(tally, fam, f"{run} part[{c}] (tiles {t0}..{t1})", part[c], g_c, (L + nchunk + 2) * R.U * (a_c + f_c))
        g_all += g_c
        a_all += a_c
        f_all += f_c
    # sum over chunks of (L_c + 2) u (A_c + F_c), plus the NCHUNK fp32 additions of the reduction
    _wgrad_entries(tally, fam, f"{run} gradient", grad, g_all, (L_max + nchunk + 2) * R.U * (a_all + f_all))
    pad = R.pad_mask("cuda")
    tally.exact(f"{run} padding of the flat gradient", grad[pad] == 0)
    return int(nz.sum()), L_max


def _wgrad_entries(tally, fam, what, got, want, bound):
    err = (got.double() - want).abs()
    ratio = torch.where(err > 0, err / bound, torch.zeros_like(err))
    tally.add(fam, what, err <= bound, torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf))


@pytest.mark.parametrize("kind", ["init", "dead"])
@pytest.mark.parametrize("case", list(CASES))
def test_nerf_mlp_against_fp64(case, kind):
    r = _run(case, kind)
    tally = Tally()
    report = [f"{case}/{kind} n={r['n']} of {r['n_max']}"]
    if r["n"] == 0:
        tally.exact("out untouched", _bits(r["out"]) == SENTINEL)
        for run, (_, scratch, grad) in r["runs"].items():
            tally.exact(f"{run} gradient of no rows", grad == 0)
        assert not tally.fails, tally.fails
        return
    dead, sv = _check_forward(r, tally)
    report.append("dead ReLUs per trunk layer " + " ".join(f"{d:.2f}" for d in dead))
    if kind == "dead" and r["n"] >= 128:
        assert sum(dead) / 8 > 0.5 and max(dead) < 0.999, dead
    for run, fam in (("dense", "wgrad-dense"), ("probe", "wgrad-probe")):
        nrows, L = _check_backward(r, run, sv, tally, fam)
        report.append(f"{run}: {nrows} rows with a gradient, at most {L} a chunk")
    report.append("worst err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(tally.worst.items())))
    print("[nerf-mlp-fp64] " + "; ".join(report))
    assert not tally.fails, tally.fails[:12]


def test_rn16_on_the_device_is_numpy_rounding():
    rng = np.random.default_rng(1)
    ys = np.concatenate([rng.standard_normal(200000) * 10.0 ** rng.uniform(-9, 5, 200000),
                         (rng.integers(2 ** 10, 2 ** 11, 50000) + 0.5) * 2.0 ** rng.integers(-24, 5, 50000)])
    got = R.rn16(torch.from_numpy(ys).cuda()).cpu().numpy()
    assert np.array_equal(got, R.numpy_rn16(ys))
