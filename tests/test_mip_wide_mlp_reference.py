"""The Mip-NeRF network kernels at 16 IPE degrees (csrc/mip_mlp_wide.cu: nerf_mlp.cuh at 12 encoder groups) against float64, layer by
layer, at multicam.py's training batch size, with a bound on every entry.

At 12 groups the kernels take paths the 8-group layout never reaches: the forward streams the skip layer as two K-chunks (the 96
encoding columns, then h4 from column 96), every saved group past the encoding moves by 4 groups (320 a tile), and the weight-gradient
jobs of layers 0 (96 columns) and 5 (352) end partway through a 128-column job.  The checks are those of test_nerf_mlp_reference.py on
the 12-group column map of tests/nerf_mlp_ref.py (Layout(12)), each from the kernel's own fp16 operands:
- encoding: the 12 saved groups equal ops.mip_encode(..., degs=16).half() bit for bit, and are a rounding of the float64 IPE within the
  per-degree bound of nerf_mlp_ref.ipe64; the view groups within 2 fp32 ulps of float64 sin / cos; rows at or past the row count encode
  a zero Gaussian ([0 x 48, 1 x 48]) and a zero view direction;
- forward, per layer (the skip layer's two K-chunks as one 352-term product), and both columns groups of `out`; rows of `out` at or past
  the row count keep their sentinel;
- dgrad, per layer from the kernel's dY of the layer above, exactly zero under dead ReLUs, the heads [drgb, 0] and [dalpha, 0 x 15]
  exact, rows at or past the row count zero;
- wgrad: every entry of every chunk's part[c] against the float64 sum over exactly that chunk's tiles, then the reduced gradient; the
  padding of the flat gradient exactly zero;
- a repeated backward is bit-identical, scratch included.
The scratch and the saved blocks start filled with NaN bytes, so an entry no kernel writes fails its check.

Cases: the network part of one MipRunner.train_step under multicam_cfg (3072 rays x 128 samples x 2 levels = 786 432 rows through one
backward: 6144 tiles, 768 a chunk) on the in-memory multiscale stand-in at its four resolutions, with the reference initialisation, the
same weights doubled with biases lowered by 0.4, and the weights after 300 fused training steps; 1, 127, 128, 129, 896 and 3700 rows of
one level; and no rows.  Every case runs a dense backward and a probe backward whose output gradient is zero except one row per tile,
the last tile and 16 random rows: with 98 k live rows a chunk the dense bound is a loose 2^-7 of sum |dY x|, the probe's about 2^-14.

Worst error / bound over all cases on an H100 (80 GB HBM3, 700 W power limit), the run prints them per case: forward 0.018, IPE 0.077
(multicam radii 1.0e-3 .. 8.3e-3 and resampled fine intervals included), view encoding 0.42, dgrad 0.045, dense wgrad 0.057, probe wgrad
0.20.  In the multicam step 0.95 M (reference weights) to 1.4 M (trained weights) of the 3.1 M output-gradient entries are fp16
subnormals.  The file takes about 24 s there, 300 training steps included, with a peak of 15 GiB of device memory in the multicam step:
4 GB of saved activations and two 4 GB scratch buffers for the repeated dense backward."""
import time

import pytest
import torch

import nerf_mlp_ref as R
from test_nerf_mlp_reference import BLOCK, SENTINEL, Tally, _bits, _probe, _tiles, _wgrad_entries

pytestmark = pytest.mark.gpu

L = R.L12
DEGS = 16
BT = BLOCK // R.ROWS               # tiles per float64 block
NAN8 = 0xFF                        # a byte every fp16 / fp32 NaN pattern of the unwritten buffers is made of
STEP_RAYS, STEP_S = 3072, 128      # multicam_cfg: batch_size 3072, num_samples 128, two levels
SIZES = {"n1": (1, 1), "n127": (1, 127), "n128": (1, 128), "n129": (3, 43), "n896": (7, 128), "n3700": (37, 100)}   # rays x samples


def _weights(kind, seed=4):
    from jnerf_b200.plugin import mip, nerf
    ref = nerf.init_reference_params(torch.Generator(device="cuda").manual_seed(seed), mip.ref_layers(DEGS), mip.REF_ORDER)
    if kind == "dead":
        ref = {k: (2 * W, b - 0.4) for k, (W, b) in ref.items()}
    return mip.pack(ref, DEGS)


def _rays(n_rays, seed):
    """Rays towards the origin with the radii of four resolutions (1.2e-3 x 1, 2, 4, 8), near 2, far 6"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    o = (torch.rand((n_rays, 3), device="cuda", generator=g) - 0.5) * 8
    d = torch.nn.functional.normalize(-o + torch.randn((n_rays, 3), device="cuda", generator=g) * 0.3, dim=-1)
    d = d * (1 + torch.rand((n_rays, 1), device="cuda", generator=g))
    radius = 1.2e-3 * 2.0 ** (torch.arange(n_rays, device="cuda") % 4).float()[:, None]
    return torch.cat([o, d, torch.nn.functional.normalize(d, dim=-1), radius, torch.full((n_rays, 1), 2.0, device="cuda"),
                      torch.full((n_rays, 1), 6.0, device="cuda")], -1).contiguous()


def _nan_bytes(nbytes):
    return torch.full((nbytes,), NAN8, dtype=torch.uint8, device="cuda")


def _encodings(rays, t, n_level):
    """enc(r0, r1) -> (fp16 encoding the kernel must save, (float64 IPE, bound), (float64 view encoding, bound)) of saved rows [r0, r1),
    which lie in one level; level k holds rows [k n_level, (k + 1) n_level) and fenceposts t[k R : (k + 1) R]."""
    from jnerf_b200 import ops
    n_rays, S = rays.shape[0], t.shape[1] - 1

    def enc(r0, r1):
        k = r0 // n_level
        a, b = r0 - k * n_level, r1 - k * n_level
        tk = t[k * n_rays:(k + 1) * n_rays]
        m = max(0, min(n_level, b) - a)
        rows = b - a
        e16 = torch.zeros((rows, 6 * DEGS), dtype=torch.float16, device="cuda")
        y = torch.zeros((rows, 6 * DEGS), dtype=torch.float64, device="cuda")
        e16[:, 3 * DEGS:], y[:, 3 * DEGS:] = 1, 1                  # rows past the row count: sin 0, cos 0 of a zero Gaussian
        e = torch.zeros_like(y)
        vx = torch.zeros((rows, 3), dtype=torch.float32, device="cuda")
        if m:
            g0, g1 = a // S, -(-(a + m) // S)
            off = a - g0 * S
            e32 = ops.mip_encode(rays[g0:g1], tk[g0:g1], degs=DEGS)[0]
            e16[:m] = e32[off:off + m].half()
            yy, ee = R.ipe64(rays[g0:g1], tk[g0:g1], "cone", True, DEGS)
            y[:m], e[:m] = yy[off:off + m], ee[off:off + m]
            vx[:m] = rays[g0:g1, 6:9].repeat_interleave(S, 0)[off:off + m]
        return e16, (y, e), R.freq_encoding(vx, 4)
    return enc


# ---------------------------------------------------------------------------------------------------------------- checks
def _check_forward(c, tally, per_degree):
    n, P, T = c["n"], c["P"], _tiles(c["n"])
    dead = torch.zeros(8, dtype=torch.float64, device="cuda")
    for t0 in range(0, T, BT):
        t1 = min(t0 + BT, T)
        r0, r1 = t0 * R.ROWS, t1 * R.ROWS
        s = R.decode(c["saved"], L.S_GROUPS, t1, t0)
        e16, (y, e), (vy, ve) = c["enc"](r0, r1)
        got = s[:, L.ENC:L.ENC + 6 * DEGS]
        tally.exact("saved encoding = mip_encode(..., degs=16).half()", _bits(got) == _bits(e16))
        ok, ratio = R.check_rounding(got, y, e)
        tally.add("ipe", "saved encoding against the float64 IPE", ok, ratio)
        per_degree.copy_(torch.maximum(per_degree, ratio.view(-1, 2, DEGS, 3).amax((0, 1, 3))))
        tally.add("view", "saved view encoding", *R.check_rounding(s[:, L.DIR:L.DIR + 32], vy, ve))
        tally.exact("saved view encoding padding", _bits(s[:, L.DIR + 27:L.DIR + 32]) == 0)
        m = max(0, min(n, r1) - r0)
        for l in range(11):
            W, b = R.layer_params(P, l, L)
            x = R.layer_input(s, l, L)
            for w0, nr, (dst, col), relu in L.FWD[l]:
                y, e = R.fwd_layer(x, W[w0:w0 + nr], b[w0:w0 + nr])
                if dst == "saved":
                    tally.add("forward", f"layer {l} rows {w0}+{nr}", *R.check_rounding(s[:, col:col + nr], y, e, relu))
                else:
                    tally.add("forward", f"layer {l} -> out[:, {col}:{col + nr}]", *R.check_rounding(c["out"][r0:r0 + m, col:col + nr], y[:m], e[:m]))
        for l in range(8):
            dead[l] += (s[:m, L.H(l):L.H(l) + 256] <= 0).double().sum()
    if c["tail"] is not None:
        tally.exact("out rows past the row count", _bits(c["tail"]) == SENTINEL)
    return (dead / max(n, 1) / 256).tolist()


def _nchunk(n):
    from jnerf_b200 import ops
    rest = ops.mip_workspace_bytes(n, DEGS)[1] - _tiles(n) * R.D_GROUPS * R.GB
    assert rest > 0 and rest % (L.N_PARAMS * 4) == 0
    return rest // (L.N_PARAMS * 4)


def _check_backward(c, run, dout, scratch, grad, tally, fam):
    n, P, T = c["n"], c["P"], _tiles(c["n"])
    nchunk = _nchunk(n)
    dys_bytes = T * R.D_GROUPS * R.GB
    part = scratch[dys_bytes:dys_bytes + nchunk * L.N_PARAMS * 4].view(torch.float32).view(nchunk, L.N_PARAMS)
    nz = (dout[:n] != 0).any(1)
    Ws = [R.layer_params(P, l, L)[0] for l in range(11)]
    g_all = torch.zeros(L.N_PARAMS, dtype=torch.float64, device="cuda")
    a_all, f_all = torch.zeros_like(g_all), torch.zeros_like(g_all)
    L_max = 0
    for ch in range(nchunk):
        c0, c1 = ch * T // nchunk, (ch + 1) * T // nchunk
        g_c, a_c, f_c = torch.zeros_like(g_all), torch.zeros_like(g_all), torch.zeros_like(g_all)
        for t0 in range(c0, c1, BT):
            t1 = min(t0 + BT, c1)
            r0, r1 = t0 * R.ROWS, t1 * R.ROWS
            d = R.decode(scratch[:dys_bytes], R.D_GROUPS, t1, t0)
            s = R.decode(c["saved"], L.S_GROUPS, t1, t0)
            m = max(0, min(n, r1) - r0)
            # dgrad, per layer from the kernel's own dY of the layer above
            head = torch.zeros((r1 - r0, R.DYS_COLS - R.DY(10)), dtype=torch.float16, device="cuda")
            head[:m, :3] = dout[r0:r0 + m, :3]
            tally.exact(f"{run} dY10 = [drgb, 0]", _bits(d[:, R.DY(10):]) == _bits(head))
            a8 = torch.zeros((r1 - r0, 16), dtype=torch.float16, device="cuda")
            a8[:m, 0] = dout[r0:r0 + m, 3]
            tally.exact(f"{run} layer-8 dY = [dalpha, 0 x 15, ..]", _bits(d[:, R.DY(8):R.DY(8) + 16]) == _bits(a8))
            tally.exact(f"{run} layer-8 dY tail", _bits(d[:, R.DY(8) + 272:R.DY(9)]) == 0)
            for l, k0, nc, mask, dst in L.DGRAD:
                y, e = R.dgrad_layer(d[:, R.DY(l):R.DY(l) + R.OUT[l]], Ws[l][:, k0:k0 + nc])
                got = d[:, dst:dst + nc]
                ok, ratio = R.check_rounding(got, y, e)
                if mask is not None:
                    live = s[:, mask:mask + nc] > 0
                    tally.exact(f"{run} layer {l} dgrad under dead ReLUs", _bits(got)[~live] == 0)
                    ok, ratio = ok | ~live, torch.where(live, ratio, torch.zeros_like(ratio))
                tally.add("dgrad", f"{run} layer {l} dgrad", ok, ratio)
            tally.exact(f"{run} dys rows past the row count", _bits(d[m:]) == 0)
            g, a, f = R.wgrad_flat(d, s, L)
            g_c += g
            a_c += a
            f_c = torch.maximum(f_c, f)
        Lc = int(nz[c0 * R.ROWS:c1 * R.ROWS].sum())
        L_max = max(L_max, Lc)
        _wgrad_entries(tally, fam, f"{run} part[{ch}] (tiles {c0}..{c1})", part[ch], g_c, (Lc + nchunk + 2) * R.U * (a_c + f_c))
        g_all += g_c
        a_all += a_c
        f_all += f_c
    _wgrad_entries(tally, fam, f"{run} gradient", grad, g_all, (L_max + nchunk + 2) * R.U * (a_all + f_all))
    tally.exact(f"{run} padding of the flat gradient", grad[R.pad_mask("cuda", L)] == 0)
    return int(nz.sum()), L_max


def _backwards(c, dout, tally, report):
    """The dense backward twice (bit-identical, scratch included), then the probe backward, each into NaN-filled scratch."""
    from jnerf_b200 import ops
    n, P = c["n"], c["P"]
    need = ops.mip_workspace_bytes(n, DEGS)[1]
    sa, sb = _nan_bytes(need), _nan_bytes(need)
    ga = ops.mip_bwd(P, c["saved"], dout, DEGS, scratch=sa)
    gb = ops.mip_bwd(P, c["saved"], dout, DEGS, scratch=sb)
    tally.exact("repeated dense backward: gradient", ga.view(torch.int32) == gb.view(torch.int32))
    tally.exact("repeated dense backward: scratch", sa == sb)
    del sb
    nrows, Lm = _check_backward(c, "dense", dout, sa, ga, tally, "wgrad-dense")
    report.append(f"dense: {nrows} rows with a gradient, at most {Lm} a chunk")
    probe = _probe(dout, max(n, 1), n)
    sa.fill_(NAN8)
    gp = ops.mip_bwd(P, c["saved"], probe, DEGS, scratch=sa)
    nrows, Lm = _check_backward(c, "probe", probe, sa, gp, tally, "wgrad-probe")
    report.append(f"probe: {nrows} rows with a gradient, at most {Lm} a chunk")


def _finish(name, c, tally, report, per_degree, t_start):
    report.append("worst err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(tally.worst.items())))
    report.append("ipe per degree " + " ".join(f"{float(v):.2f}" for v in per_degree))
    report.append(f"{time.time() - t_start:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    print(f"[mip-wide-fp64] {name} n={c['n']}; " + "; ".join(report))
    assert not tally.fails, tally.fails[:12]


# ---------------------------------------------------------------------------------------------------------------- multicam step
def _multicam_runner(tmp, batch, **over):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.mip_runner import MipRunner, multicam_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**multicam_cfg(seed=7, log_dir=str(tmp), using_fp16=True, **over))
    cfg = get_cfg()
    for split in ("train", "val", "test"):
        cfg.dataset[split].update(n_images=4, H=400, W=400)
    cfg.dataset.train.batch_size = batch
    return MipRunner()


@pytest.fixture(scope="module")
def step(tmp_path_factory):
    """(a multicam_cfg runner at batch 3072, the weights of a stand-in runner after 300 fused training steps of 1024 rays)"""
    tmp = tmp_path_factory.mktemp("mip_wide")
    sched = dict(optim=dict(type="Adam", lr=2e-3, eps=1e-15, betas=(0.9, 0.99)),
                 linearlog=dict(type="LinearLog", end_lr=2e-4, max_steps=300, lr_delay_steps=0, lr_delay_mult=1.0))
    tr = _multicam_runner(tmp / "train", 1024, **sched)
    tr.train(300)
    trained = tr.model.params.detach().clone()
    del tr
    torch.cuda.empty_cache()
    return _multicam_runner(tmp / "step", STEP_RAYS), trained


@pytest.mark.parametrize("kind", ["init", "dead", "trained"])
def test_multicam_step_against_fp64(step, kind):
    """MipRunner.train_step's network part: both levels' forwards into the runner's saved buffer (_forward_levels), the loss gradient of
    both levels with the batch's lossmult mask and grad_scale = R, one backward over 786 432 rows."""
    from jnerf_b200 import ops
    t_start = time.time()
    torch.cuda.reset_peak_memory_stats()
    r, trained = step
    P = trained if kind == "trained" else _weights(kind)
    r.model.params.data.copy_(P)
    rays, target, lossmult = next(r.dataset["train"])
    assert rays.shape[0] == STEP_RAYS and r.sampler.num_samples == STEP_S
    n_level = STEP_RAYS * STEP_S
    r._saved = _nan_bytes(2 * ops.mip_workspace_bytes(n_level, DEGS)[0])   # every saved group must be written
    t, raw = r._forward_levels(rays, save=True)
    s = r.sampler
    _, _, draw = ops.mip_composite_loss_bwd(raw, t, rays, target, lossmult, s.rgb_padding, s.density_bias, s.white_bkgd, r.coarse_loss_mult,
                                            grad_scale=float(STEP_RAYS))
    torch.cuda.synchronize()
    c = dict(n=2 * n_level, P=r.model.params.detach(), out=raw, tail=None, saved=r._saved, enc=_encodings(rays, t, n_level))
    sub = int(((draw != 0) & (draw.abs() < 2.0 ** -14)).sum())
    report = [f"lossmult {sorted(set(lossmult.tolist()))}, radii {float(rays[:, 9].min()):.2e} .. {float(rays[:, 9].max()):.2e}",
              f"{sub} of {draw.numel()} output-gradient entries fp16-subnormal, {int((draw == 0).sum())} zero"]
    tally, per_degree = Tally(), torch.zeros(DEGS, dtype=torch.float64, device="cuda")
    dead = _check_forward(c, tally, per_degree)
    report.append("dead ReLUs per trunk layer " + " ".join(f"{d:.2f}" for d in dead))
    if kind == "dead":
        assert sum(dead) / 8 > 0.5 and max(dead) < 0.999, dead
    _backwards(c, draw.contiguous(), tally, report)
    r._saved = None
    _finish(f"multicam step/{kind}", c, tally, report, per_degree, t_start)


# ---------------------------------------------------------------------------------------------------------------- small sizes
@pytest.mark.parametrize("kind", ["init", "dead"])
@pytest.mark.parametrize("case", list(SIZES))
def test_row_counts_against_fp64(case, kind):
    """One level of n_rays x n_samples rows (a partial last tile, fewer tiles than chunks): `out` is a view into a larger buffer whose
    rows past n must keep their sentinel."""
    from jnerf_b200 import ops
    t_start = time.time()
    torch.cuda.reset_peak_memory_stats()
    n_rays, S = SIZES[case]
    n = n_rays * S
    P = _weights(kind)
    rays = _rays(n_rays, seed=n)
    t = ops.mip_sample(rays, S, False, True, ops.pcg32_seed(n))
    big = torch.empty((n + 300, 4), dtype=torch.float16, device="cuda")
    big.view(torch.int16).fill_(SENTINEL)
    saved = _nan_bytes(ops.mip_workspace_bytes(n, DEGS)[0])
    ops.mip_fwd(rays, t, P, out=big[:n], saved=saved, degs=DEGS)
    dout = (torch.randn((n, 4), device="cuda", generator=torch.Generator(device="cuda").manual_seed(n)) * 0.1).half()
    c = dict(n=n, P=P, out=big[:n], tail=big[n:], saved=saved, enc=_encodings(rays, t, n))
    tally, per_degree, report = Tally(), torch.zeros(DEGS, dtype=torch.float64, device="cuda"), []
    dead = _check_forward(c, tally, per_degree)
    report.append("dead ReLUs per trunk layer " + " ".join(f"{d:.2f}" for d in dead))
    if kind == "dead" and n >= 128:
        assert sum(dead) / 8 > 0.5 and max(dead) < 0.999, dead
    _backwards(c, dout, tally, report)
    _finish(f"{case}/{kind}", c, tally, report, per_degree, t_start)


def test_no_rows():
    """mip_fwd of no rows leaves out and saved untouched; mip_bwd of no rows writes every chunk's part (all zero) and a zero gradient."""
    from jnerf_b200 import ops
    P = _weights("init")
    rays = _rays(4, seed=1)
    t = ops.mip_sample(rays, 128, False, True, ops.pcg32_seed(1))
    out = torch.empty((16, 4), dtype=torch.float16, device="cuda")
    out.view(torch.int16).fill_(SENTINEL)
    saved = _nan_bytes(ops.mip_workspace_bytes(128, DEGS)[0])
    ops.mip_fwd(rays[:0], t[:0], P, out=out, saved=saved, degs=DEGS)
    scratch = _nan_bytes(ops.mip_workspace_bytes(0, DEGS)[1])
    assert scratch.numel() == _nchunk(0) * L.N_PARAMS * 4
    grad = ops.mip_bwd(P, saved[:0], torch.zeros((0, 4), dtype=torch.float16, device="cuda"), DEGS, scratch=scratch)
    torch.cuda.synchronize()
    assert bool((_bits(out) == SENTINEL).all()) and bool((saved == NAN8).all())
    assert grad.shape == (L.N_PARAMS,) and bool((grad.view(torch.int32) == 0).all())
    assert bool((scratch.view(torch.int32) == 0).all())
