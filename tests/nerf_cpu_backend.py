"""The vanilla NeRF operators of jnerf_b200/ops.py (nerf_fwd / nerf_density / nerf_bwd) as an fp32 torch restatement on CPU tensors,
installed on top of tests/cpu_backend.py so that the host logic around them -- OriginNeRFNetworks' autograd function, the occupancy
update through model.density, the optimizer over the flat parameter vector, checkpoints -- runs without a GPU.  Test infrastructure,
like cpu_backend: the kernels themselves are checked against the same chain by tests/test_nerf_gpu.py."""
import torch

import cpu_backend


def _chain(flat, pos, dirs=None):
    """ori_nerf_network.py:34-67 in fp32 on the fp16-rounded encodings: (n, 4) {rgb, alpha}, or alpha (n,) when dirs is None."""
    from jnerf_b200.plugin import nerf
    ref = nerf.unpack(flat) if not isinstance(flat, dict) else flat
    enc = nerf.freq_encode(pos.float(), 10).half().float()
    lin = lambda name, x: x @ ref[name][0].t() + ref[name][1]
    h = enc
    for i in range(8):
        h = torch.relu(lin(f"pts_linears.{i}", h))
        if i == 4:
            h = torch.cat([enc, h], -1)
    alpha = lin("alpha_linear", h)
    if dirs is None:
        return alpha[:, 0]
    encd = nerf.freq_encode(dirs.float(), 4).half().float()
    v = torch.relu(lin("views_linears.0", torch.cat([lin("feature_linear", h), encd], -1)))
    return torch.cat([lin("rgb_linear", v), alpha], -1)


def install(monkeypatch, fake=None):
    """cpu_backend.install (unless `fake` is the OracleOps it returned) + the NeRF operators, logged in the same call list."""
    if fake is None:
        fake = cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops
    from jnerf_b200.plugin import nerf

    def nerf_fwd(coords, params, n_dev=None, save=False, out=None):
        fake._log("nerf_fwd")
        n = coords.shape[0]
        live = cpu_backend._live(n_dev, n)
        if out is None:
            out = torch.empty((n, 4), dtype=torch.float16)
        with torch.no_grad():
            out[:live] = _chain(params, coords[:live, :3], coords[:live, 4:7]).half()
        return out, ((coords[:live].clone(), live) if save else None)

    def nerf_density(pos, params):
        fake._log("nerf_density")
        with torch.no_grad():
            return _chain(params, pos).half()

    def nerf_bwd(params, saved, dout, n_dev=None):
        fake._log("nerf_bwd")
        coords, live = saved
        live = cpu_backend._live(n_dev, live)
        ref = {k: (W.requires_grad_(), b.requires_grad_()) for k, (W, b) in nerf.unpack(params).items()}
        with torch.enable_grad():
            (_chain(ref, coords[:live, :3], coords[:live, 4:7]) * dout[:live].float()).sum().backward()
        grad = torch.zeros(params.numel(), dtype=torch.float32)
        for name, (W, b) in ref.items():
            Wk, bk, cols = nerf._kernel_views(grad, name)
            for rc, kc, n in cols:
                Wk[:, kc:kc + n] = W.grad[:, rc:rc + n]
            bk.copy_(b.grad)
        return grad

    for name, fn in (("nerf_fwd", nerf_fwd), ("nerf_density", nerf_density), ("nerf_bwd", nerf_bwd),
                     ("nerf_param_count", lambda: nerf.N_PARAMS)):
        monkeypatch.setattr(real_ops, name, fn)
    return fake
