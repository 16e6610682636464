"""Test infrastructure: run the HOST logic of the product (plugin classes, Runner, checkpoints, data-parallel bookkeeping) on a
machine without a GPU by swapping the C-ABI operator layer (`jnerf_b200.ops`, i.e. libngp_b200.so's kernels) for the oracle
(oracle/ngp_oracle.c through tests/oracle_lib.py) and mapping torch's "cuda" device to "cpu".

This is NOT a CPU fallback of the product: it lives under tests/, is installed only through the `cpu_backend` fixture, and exists
so that the Python glue around the kernels (call order, buffer aliasing, RNG stream bookkeeping, adaptive ray batch, optimizer
step order, checkpoint formats, tiled rendering) is exercised by `pytest -m "not gpu"` every round.  The kernels themselves are
checked against the same oracle by the `-m gpu` tests."""
import types

import numpy as np
import torch

import oracle_lib as ol

_FACTORIES = ["zeros", "empty", "ones", "full", "rand", "randn", "randperm", "tensor", "arange", "zeros_like", "empty_like", "ones_like",
              "as_tensor", "randint", "linspace"]


def _cpu_dev(d):
    if d is None:
        return None
    if isinstance(d, torch.device):
        return torch.device("cpu") if d.type == "cuda" else d
    if isinstance(d, str) and d.startswith("cuda"):
        return "cpu"
    return d


def _np(t, dtype=None):
    a = t.detach().cpu().numpy()
    return np.ascontiguousarray(a if dtype is None else a.astype(dtype, copy=False))


def _u32view(t):
    return _np(t).view(np.uint32)


class CpuHashLevels:
    """ops.HashLevels without the device table: the offsets come from the real host entry point (ngp_hash_offsets)."""

    def __init__(self, aabb_scale=1, n_levels=16, base_resolution=16, log2_hashmap_size=19, device="cpu", primes=(1, 19349663, 83492791)):
        assert tuple(primes) == (1, 19349663, 83492791), "the CPU stand-in evaluates the configs' hash only"
        self.primes = tuple(primes)
        self.cfg = ol.HashCfg(aabb_scale, n_levels, base_resolution, log2_hashmap_size)
        self.n_levels, self.base_resolution = n_levels, base_resolution
        self.offsets = self.cfg.offsets
        self.per_level_scale = self.cfg.per_level_scale
        self.log2_per_level_scale = float(self.cfg.log2_pls)
        self.n_entries, self.n_params = self.cfg.n_entries, self.cfg.n_params
        self.table = torch.zeros(n_levels * 32, dtype=torch.uint8)


def _live(n_dev, n):
    return n if n_dev is None else min(int(n_dev.reshape(-1)[0].item()), n)


class OracleOps:
    """Same function names and signatures as jnerf_b200/ops.py, computed by the oracle on CPU tensors."""

    F32, F16 = 0, 1
    HashLevels = CpuHashLevels
    calls = None            # list of op names in call order (tests assert on the sequence)

    def __init__(self):
        self.calls = []
        import jnerf_b200.lib as real_lib
        self.lib = real_lib                     # host-only helpers (workspace sizes, pcg32) still come from the real library

    def _log(self, name):
        self.calls.append(name)

    # ---- encoders / MLP ------------------------------------------------------------------------------------
    def hash_fwd(self, x, grid, levels):
        self._log("hash_fwd")
        out = ol.hash_fwd(levels.cfg, _np(x, np.float32), _np(grid), acc32=grid.dtype == torch.float16)
        return torch.from_numpy(out)

    def hash_bwd(self, x, dy, levels, grid_grad=None):
        self._log("hash_bwd")
        g = ol.hash_bwd(levels.cfg, _np(x, np.float32), _np(dy), acc32=dy.dtype == torch.float16)
        g = torch.from_numpy(g)
        if grid_grad is not None:
            grid_grad.copy_(g)
            return grid_grad
        return g

    def sh_fwd(self, dirs, dtype=torch.float16):
        self._log("sh_fwd")
        return torch.from_numpy(ol.sh(_np(dirs, np.float32), np.float16 if dtype == torch.float16 else np.float32))

    def mlp_fwd(self, W, X, n_hidden_matmuls, save_inter=True):
        self._log("mlp_fwd")
        Y, inter = ol.mlp_fwd(_np(W), _np(X), n_hidden_matmuls)
        return torch.from_numpy(Y), (torch.from_numpy(inter) if save_inter else None)

    def mlp_bwd(self, W, X, inter, dY, n_hidden_matmuls, n_out_valid, need_dx=True, need_temps=False):
        self._log("mlp_bwd")
        dX, temps, dW = ol.mlp_bwd(_np(W), _np(X), _np(inter), _np(dY), n_hidden_matmuls, n_out_valid)
        return (torch.from_numpy(dX) if need_dx else None), (torch.from_numpy(temps) if need_temps else None), torch.from_numpy(dW)

    # ---- fused network -------------------------------------------------------------------------------------
    def network_fwd(self, coords, grid, levels, wd, wr, n_dev=None, save_enc=True, out=None, enc=None):
        self._log("network_fwd")
        n = coords.shape[0]
        live = _live(n_dev, n)
        if out is None:
            out = torch.zeros((n, 4), dtype=torch.float16)
        if enc is None and save_enc:
            enc = torch.zeros((n, 32), dtype=torch.float16)
        if live:
            c = _np(coords[:live], np.float32)
            o, e, _ = ol.network_fwd(levels.cfg, c[:, :3].copy(), c[:, 4:].copy(), _np(grid), _np(wd), _np(wr), acc32=True)
            out[:live] = torch.from_numpy(o)
            if enc is not None:
                enc[:live] = torch.from_numpy(e)
        return out, enc

    def network_bwd(self, coords, enc, levels, wd, wr, dout, grid_grad, dwd, dwr, n_dev=None):
        self._log("network_bwd")
        live = _live(n_dev, coords.shape[0])
        if not live:
            return
        c = _np(coords[:live], np.float32)
        pos, dirs = c[:, :3].copy(), c[:, 4:].copy()
        e, Wd, Wr, d = _np(enc[:live]), _np(wd), _np(wr), _np(dout[:live]).astype(np.float32)
        h, inter_d = ol.mlp_fwd(Wd, e, 0)
        rin = np.concatenate([h, ol.sh(dirs, np.float16)], 1)
        _, inter_r = ol.mlp_fwd(Wr, rin, 1)
        dYr = np.zeros((live, 16), np.float16)
        dYr[:, :3] = d[:, :3]
        d_rin, _, dWr = ol.mlp_bwd(Wr, rin, inter_r, dYr, 1, 3)
        dYd = d_rin[:, :16].astype(np.float32)
        dYd[:, 0] += d[:, 3]                                                   # + dL/dsigma (ngp_network.py:83)
        d_enc, _, dWd = ol.mlp_bwd(Wd, e, inter_d, dYd.astype(np.float16), 0, 16)
        g = ol.hash_bwd(levels.cfg, pos, d_enc, acc32=True)
        grid_grad += torch.from_numpy(g).to(grid_grad.dtype)                   # ACCUMULATED, like the kernel (caller zeroes)
        dwd += torch.from_numpy(dWd)
        dwr += torch.from_numpy(dWr)

    def density_fwd(self, pos, grid, levels, wd):
        self._log("density_fwd")
        e = ol.hash_fwd(levels.cfg, _np(pos, np.float32), _np(grid), acc32=True)
        Y, _ = ol.mlp_fwd(_np(wd), e, 0)
        return torch.from_numpy(np.ascontiguousarray(Y[:, 0]))

    # ---- sampler -------------------------------------------------------------------------------------------
    def march(self, rays_o, rays_d, bitfield, aabb, max_samples, cone_angle, near, cascades, const_dt, rng, coords=None, workspace=None):
        self._log("march")
        c, ray_idx, numsteps, counters = ol.march(_np(rays_o, np.float32), _np(rays_d, np.float32), _np(bitfield), aabb, max_samples, cone_angle, near,
                                                  cascades, const_dt, rng)
        total = min(int(counters[1]), max_samples)
        if coords is None:
            coords = torch.zeros((max_samples, 7), dtype=torch.float32)
        coords[:total] = torch.from_numpy(c[:total])                           # rows beyond the total keep their old content, as on the GPU
        return coords, torch.from_numpy(ray_idx.view(np.int32)), torch.from_numpy(numsteps.view(np.int32)), torch.from_numpy(counters.view(np.int32))

    def compact(self, coords, numsteps, max_compacted, alias=False, zero_fill=True):
        self._log("compact")
        out, ns, cnt = ol.compact(_np(coords, np.float32), _u32view(numsteps), max_compacted)
        ns, cnt = torch.from_numpy(ns.view(np.int32)), torch.from_numpy(cnt.view(np.int32))
        return (coords if alias else torch.from_numpy(out)), ns, cnt

    def composite_fwd(self, net, coords, numsteps_in, numsteps_c, bg, cascades=5):
        self._log("composite_fwd")
        return torch.from_numpy(ol.composite_fwd(_np(net), _np(coords, np.float32), _u32view(numsteps_in), _u32view(numsteps_c), _np(bg), cascades))

    def composite_bwd(self, net, coords, numsteps_c, loss_grad, rgb_ray, mean, cascades=5):
        self._log("composite_bwd")
        return torch.from_numpy(ol.composite_bwd(_np(net), _np(coords, np.float32), _u32view(numsteps_c), _np(loss_grad), _np(rgb_ray),
                                                 float(mean.reshape(-1)[0]), cascades))

    def composite_infer(self, net, coords, numsteps, cascades=5):
        self._log("composite_infer")
        rgb, alpha = ol.composite_infer(_np(net), _np(coords, np.float32), _u32view(numsteps), cascades)
        return torch.from_numpy(rgb), torch.from_numpy(alpha)

    def composite_loss_bwd(self, net, coords, numsteps_in, numsteps_c, bg, target, mean, delta=0.1, cascades=5, dnet=None, rgb=None, loss=None,
                           reg_scale=1.0):
        self._log("composite_loss_bwd")
        ol.oracle().orc_set_reg_scale(float(reg_scale))
        R = numsteps_c.shape[0]
        n, c, ns_in, ns_c = _np(net), _np(coords, np.float32), _u32view(numsteps_in), _u32view(numsteps_c)
        r = ol.composite_fwd(n, c, ns_in, ns_c, _np(bg), cascades)
        g, l = ol.huber_grad(r, _np(target), delta)
        d = ol.composite_bwd(n, c, ns_c, g.reshape(R, 3), r, float(mean.reshape(-1)[0]), cascades)
        ol.oracle().orc_set_reg_scale(1.0)
        rows = int((ns_c[:, 0].astype(np.int64)).sum())
        if dnet is None:
            dnet = torch.zeros_like(net)
        dnet[:rows] = torch.from_numpy(d[:rows])                              # rows not covered by a ray are not written (see the kernel)
        return torch.from_numpy(r), torch.from_numpy(l.reshape(R, 3).sum(1)), dnet

    # ---- occupancy grid ------------------------------------------------------------------------------------
    def grid_mark_untrained(self, grid, focal, xforms, res):
        self._log("grid_mark_untrained")
        g = _np(grid)
        ol.mark_untrained(g, _np(focal), _np(xforms), res)
        grid.copy_(torch.from_numpy(g))

    def grid_generate_samples(self, n, rng, step_dev, aabb, grid, n_cascades, thresh):
        self._log("grid_generate_samples")
        pos, idx = ol.generate_grid_samples(n, rng, int(step_dev.reshape(-1)[0]), aabb, _np(grid), n_cascades, thresh)
        return torch.from_numpy(pos), torch.from_numpy(idx.view(np.int32))

    def grid_splat(self, indices, mlp_out, grid_tmp):
        self._log("grid_splat")
        g = _np(grid_tmp)
        ol.splat(_u32view(indices), _np(mlp_out), g)
        grid_tmp.copy_(torch.from_numpy(g))

    def grid_ema(self, grid, grid_tmp, decay=0.95):
        self._log("grid_ema")
        g = _np(grid)
        ol.ema(g, _np(grid_tmp), decay)
        grid.copy_(torch.from_numpy(g))

    def grid_update_bitfield(self, grid, mean, bitfield, cascades=5):
        self._log("grid_update_bitfield")
        g = _np(grid)
        mu = ol.grid_mean(g)
        mean.fill_(mu)
        bits = ol.update_bitfield(g, mu, cascades)
        bitfield.copy_(torch.from_numpy(bits[:bitfield.numel()]))

    # ---- optimizer / data ----------------------------------------------------------------------------------
    def adam_ema(self, param, grad, m, v, master, lr, step, beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95, grad_scale=1.0, zero_grad=True):
        self._log("adam_ema")
        p, mm, vv, ms = _np(param).reshape(-1), _np(m), _np(v), _np(master)
        g = (_np(grad).reshape(-1).astype(np.float32) * np.float32(grad_scale)).astype(np.float32)
        ol.adam_ema(p, g, mm, vv, ms, lr, step, beta1, beta2, eps, ema_decay)
        param.copy_(torch.from_numpy(p).reshape(param.shape))
        m.copy_(torch.from_numpy(mm)); v.copy_(torch.from_numpy(vv)); master.copy_(torch.from_numpy(ms))
        if zero_grad:
            grad.zero_()

    def raygen(self, pix, W, H, xforms, focal, principal):
        self._log("raygen")
        img, o, d = ol.raygen(_u32view(pix), W, H, _np(xforms), _np(focal), _np(principal))
        return torch.from_numpy(img.view(np.int32)), torch.from_numpy(o), torch.from_numpy(d)

    def prepare_batch(self, pix, W, H, xforms, focal, principal, images, bg):
        self._log("prepare_batch")
        img, o, d = self.raygen(pix, W, H, xforms, focal, principal)
        self.calls.pop()                                                       # counted as one operator
        rgba = images.reshape(-1, 4)[pix.long()]
        rgba = rgba.float() / 255.0 if rgba.dtype == torch.uint8 else rgba.float()
        target = rgba[:, :3] * rgba[:, 3:] + bg * (1 - rgba[:, 3:])            # runner.py:68
        return img, o, d, target.contiguous()

    def blend_target(self, rgba, bg, target=None):
        self._log("blend_target")
        t = (rgba[:, :3] * rgba[:, 3:] + bg * (1 - rgba[:, 3:])).contiguous()   # runner.py:68
        if target is not None:
            target.copy_(t)
            return target
        return t

    def pcg32_seed(self, seed=1337, seq=1):
        return ol.pcg32_seed(seed, seq)

    def pcg32_advance(self, si, delta=1 << 32):
        return ol.pcg32_advance(si, delta)


def install(monkeypatch):
    # the sequential step by default (tests count one step's calls); tests of the software pipeline over steps switch it back on
    monkeypatch.setenv("NGP_PIPELINE", "0")
    """Route jnerf_b200.ops to the oracle and torch's "cuda" device to the CPU for the duration of one test."""
    import jnerf_b200.ops as real_ops
    fake = OracleOps()
    for name in dir(fake):
        if name.startswith("_") or name in ("calls", "lib"):
            continue
        monkeypatch.setattr(real_ops, name, getattr(fake, name), raising=False)
    # everything else in ops.py (dp exchange) needs the GPU: make an accidental call obvious
    for name in ("dp_exchange_step", "dp_exchange_wait", "mlp_bwd_dgrad"):
        monkeypatch.setattr(real_ops, name, lambda *a, _n=name, **k: (_ for _ in ()).throw(RuntimeError(f"{_n} has no CPU stand-in")))

    for fn in _FACTORIES:
        orig = getattr(torch, fn)

        def wrapped(*a, _orig=orig, **k):
            if "device" in k:
                k["device"] = _cpu_dev(k["device"])
            return _orig(*a, **k)
        monkeypatch.setattr(torch, fn, wrapped)
    gen = torch.Generator
    monkeypatch.setattr(torch, "Generator", lambda device=None: gen(device=_cpu_dev(device) or "cpu"))
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    to = torch.Tensor.to

    def to_cpu(self, *a, **k):
        a = tuple(_cpu_dev(x) if isinstance(x, (str, torch.device)) else x for x in a)
        if "device" in k:
            k["device"] = _cpu_dev(k["device"])
        return to(self, *a, **k)
    monkeypatch.setattr(torch.Tensor, "to", to_cpu)
    load = torch.load
    monkeypatch.setattr(torch, "load", lambda f, *a, **k: load(f, *a, **dict(k, map_location="cpu")))
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)

    class _FakeStream:                                             # the host-batch pipeline's copy stream: everything is synchronous here
        cuda_stream = 0

        def wait_event(self, ev):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    class _FakeEvent:
        def __init__(self, *a, **k):
            pass

        def record(self, *a, **k):
            pass

        def elapsed_time(self, other):
            return 1.0

        def synchronize(self):
            pass
    one = _FakeStream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: one)
    monkeypatch.setattr(torch.cuda, "Stream", _FakeStream)
    monkeypatch.setattr(torch.cuda, "stream", lambda st: st)
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, *a, **k: None)
    from jnerf_b200.plugin import dataset as D
    monkeypatch.setattr(D, "DEVICE", "cpu")
    return fake
