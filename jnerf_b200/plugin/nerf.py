"""FrequencyEncoder / OriginNeRFNetworks: mirror of models/position_encoders/freq_encoder/freq_encoder.py and
models/networks/ori_nerf_network.py (projects/nerf/configs/nerf_base.py).

With fp16=True the network runs on csrc/nerf_mlp.cu (include/ngp_b200.h F1-F4): the encoding and all eleven layers in one forward
kernel, a deterministic backward, and ONE flat fp16 parameter vector `params` in the kernels' padded layout, so that Adam + EMA is one
sweep.  With fp16=False it is a plain fp32 torch.nn.Linear chain with the reference's module names -- the reference semantics the tests
compare the kernels against.

Flat layout (DESIGN.md section 10): kernel layer l holds a weight (OUT[l], IN[l]) row-major, then a bias (OUT[l]); padding is zero.
    l 0      pts_linears.0   (256, 63)  -> columns 0..62
    l 1-4,6,7 pts_linears.l  (256, 256)
    l 5      pts_linears.5   (256, 319) -> columns 0..62 (enc_pos) and 64..319 (h4)
    l 8      alpha_linear    (1, 256)   -> row 0;  feature_linear (256, 256) -> rows 16..271
    l 9      views_linears.0 (128, 283) -> columns 0..282 (feature, then enc_dir)
    l 10     rgb_linear      (3, 128)   -> rows 0..2"""
import math

import torch

from .. import ops
from ..utils.config import get_cfg
from ..utils.registry import ENCODERS, NETWORKS, build_from_cfg
from .module import Module
from .network import invariant_uniform

IN = (64, 256, 256, 256, 256, 320, 256, 256, 256, 288, 128)
OUT = (256,) * 8 + (272, 128, 16)
W_OFF = [0]
for _o, _i in zip(OUT, IN):
    W_OFF.append(W_OFF[-1] + _o * (_i + 1))
N_PARAMS = W_OFF[-1]

# reference name -> (shape (out, in), kernel layer, first kernel row, [(first reference column, first kernel column, columns)])
REF_LAYERS = {f"pts_linears.{i}": ((256, 256), i, 0, [(0, 0, 256)]) for i in (1, 2, 3, 4, 6, 7)}
REF_LAYERS.update({
    "pts_linears.0": ((256, 63), 0, 0, [(0, 0, 63)]),
    "pts_linears.5": ((256, 319), 5, 0, [(0, 0, 63), (63, 64, 256)]),
    "views_linears.0": ((128, 283), 9, 0, [(0, 0, 283)]),
    "feature_linear": ((256, 256), 8, 16, [(0, 0, 256)]),
    "alpha_linear": ((1, 256), 8, 0, [(0, 0, 256)]),
    "rgb_linear": ((3, 128), 10, 0, [(0, 0, 128)]),
})
# construction order of the reference's modules (ori_nerf_network.py:21-26): the order the initialiser draws them in
REF_ORDER = [f"pts_linears.{i}" for i in range(8)] + ["views_linears.0", "feature_linear", "alpha_linear", "rgb_linear"]


def _kernel_views(flat, name, layers=REF_LAYERS):
    (o, _), l, r0, cols = layers[name]
    W = flat[W_OFF[l]:W_OFF[l] + OUT[l] * IN[l]].view(OUT[l], IN[l])
    b = flat[W_OFF[l] + OUT[l] * IN[l]:W_OFF[l + 1]]
    return W[r0:r0 + o], b[r0:r0 + o], cols


def pack(ref, layers=REF_LAYERS):
    """{reference name: (weight (out, in), bias (out,))} -> the flat fp16 vector of the kernels (layers: the name table, e.g. plugin/mip.py's)."""
    dev = next(iter(ref.values()))[0].device
    flat = torch.zeros(N_PARAMS, dtype=torch.float16, device=dev)
    for name, (W, b) in ref.items():
        Wk, bk, cols = _kernel_views(flat, name, layers)
        for rc, kc, n in cols:
            Wk[:, kc:kc + n] = W[:, rc:rc + n].to(torch.float16)
        bk.copy_(b.to(torch.float16))
    return flat


def unpack(flat, layers=REF_LAYERS):
    """The flat vector (parameters or gradients) -> {reference name: (weight (out, in), bias (out,))} in fp32."""
    out = {}
    for name, ((o, i), _, _, _) in layers.items():
        Wk, bk, cols = _kernel_views(flat, name, layers)
        W = torch.empty((o, i), dtype=torch.float32, device=flat.device)
        for rc, kc, n in cols:
            W[:, rc:rc + n] = Wk[:, kc:kc + n].float()
        out[name] = (W, bk.float().clone())
    return out


def init_reference_params(gen, layers=REF_LAYERS, order=REF_ORDER):
    """Jittor's nn.Linear initialisation, restated: weight invariant_uniform((out, in)), bias U(+-1/sqrt(in)); fp32."""
    ref = {}
    for name in order:
        (o, i) = layers[name][0]
        W = invariant_uniform((o, i), gen)
        b = (torch.rand(o, device="cuda", generator=gen) * 2 - 1) / math.sqrt(i)
        ref[name] = (W, b)
    return ref


def freq_encode(x, multires, include_input=True, log_sampling=True):
    """[x, sin(x f_0), cos(x f_0), ..., sin(x f_(L-1)), cos(x f_(L-1))] in fp32 (freq_encoder.py:22-45)."""
    if log_sampling:
        freqs = 2.0 ** torch.linspace(0.0, multires - 1, multires)
    else:
        freqs = torch.linspace(1.0, 2.0 ** (multires - 1), multires)
    parts = [x] if include_input else []
    for f in freqs.tolist():
        parts += [torch.sin(x * f), torch.cos(x * f)]
    return torch.cat(parts, -1)


@ENCODERS.register_module()
class FrequencyEncoder(Module):
    """freq_encoder.py:10-50.  Inside OriginNeRFNetworks with fp16=True the encoding is computed in the network's forward kernel."""

    def __init__(self, multires, include_input=True, input_dims=3, log_sampling=True):
        super().__init__()
        self.using_fp16 = bool(get_cfg().fp16)
        self.multires, self.include_input, self.input_dims, self.log_sampling = multires, include_input, input_dims, log_sampling
        self.out_dim = input_dims * (int(include_input) + 2 * multires)

    def execute(self, x):
        res = freq_encode(x.float(), self.multires, self.include_input, self.log_sampling)
        return res.half() if self.using_fp16 else res


class _NeRFFn(torch.autograd.Function):
    """OriginNeRFNetworks.execute_ (ori_nerf_network.py:34-56) as one forward kernel and the backward kernels."""

    @staticmethod
    def forward(ctx, coords, params):
        out, saved = ops.nerf_fwd(coords, params, save=True)
        ctx.save_for_backward(params)
        ctx.saved = saved
        return out

    @staticmethod
    def backward(ctx, dout):
        (params,) = ctx.saved_tensors
        grad = ops.nerf_bwd(params, ctx.saved, dout.contiguous().half())
        ctx.saved = None
        return None, grad.half()


@NETWORKS.register_module()
class OriginNeRFNetworks(Module):
    """ori_nerf_network.py:8-70 for its only configuration, D=8, W=256, skips=[4], with FrequencyEncoder(10) / FrequencyEncoder(4)."""

    def __init__(self, D=8, W=256, skips=[4]):
        super().__init__()
        self.cfg = get_cfg()
        self.using_fp16 = bool(self.cfg.fp16)
        self.pos_encoder = build_from_cfg(self.cfg.encoder.pos_encoder, ENCODERS)
        self.dir_encoder = build_from_cfg(self.cfg.encoder.dir_encoder, ENCODERS)
        if (D, W, list(skips), self.pos_encoder.out_dim, self.dir_encoder.out_dim) != (8, 256, [4], 63, 27):
            raise NotImplementedError("OriginNeRFNetworks: the kernels are built for D=8, W=256, skips=[4], FrequencyEncoder multires 10 / 4")
        self.D, self.W, self.skips = D, W, list(skips)
        gen = torch.Generator(device="cuda").manual_seed(int(self.cfg.seed or 1) + 1)
        ref = init_reference_params(gen)
        if self.using_fp16:
            self.params = torch.nn.Parameter(pack(ref))
        else:
            def linear(name):
                (o, i) = REF_LAYERS[name][0]
                lin = torch.nn.Linear(i, o).cuda()
                with torch.no_grad():
                    lin.weight.copy_(ref[name][0])
                    lin.bias.copy_(ref[name][1])
                return lin
            self.pts_linears = torch.nn.ModuleList([linear(f"pts_linears.{i}") for i in range(D)])
            self.views_linears = torch.nn.ModuleList([linear("views_linears.0")])
            self.feature_linear = linear("feature_linear")
            self.alpha_linear = linear("alpha_linear")
            self.rgb_linear = linear("rgb_linear")

    def _trunk(self, pos):
        enc = self.pos_encoder(pos)
        h = enc
        for i, lin in enumerate(self.pts_linears):
            h = torch.relu(lin(h))
            if i in self.skips:
                h = torch.cat([enc, h], -1)
        return h

    def execute(self, pos_input, dir_input):
        if self.using_fp16:
            coords = torch.zeros((pos_input.shape[0], 7), dtype=torch.float32, device=pos_input.device)
            coords[:, :3] = pos_input
            coords[:, 4:] = dir_input
            return _NeRFFn.apply(coords, self.params)
        h = self._trunk(pos_input)
        alpha = self.alpha_linear(h)
        v = torch.relu(self.views_linears[0](torch.cat([self.feature_linear(h), self.dir_encoder(dir_input)], -1)))
        return torch.cat([self.rgb_linear(v), alpha], -1)

    def density(self, pos_input):
        with torch.no_grad():
            if self.using_fp16:
                return ops.nerf_density(pos_input.contiguous(), self.params).unsqueeze(-1)
            return self.alpha_linear(self._trunk(pos_input))

    @torch.no_grad()
    def infer(self, rows, n_dev, out):
        """Inference forward on (N,7) NerfCoordinate rows into out (N,4): the renderers' network call.  n_dev (device uint32) bounds
        the rows the kernel reads and writes."""
        if self.using_fp16:
            ops.nerf_fwd(rows, self.params, n_dev=n_dev, out=out)
        else:
            out.copy_(self.execute(rows[:, :3], rows[:, 4:]))

    def reference_params(self):
        """{reference name: (weight, bias)} in fp32, e.g. pts_linears.5 -> ((256, 319), (256,))."""
        if self.using_fp16:
            return unpack(self.params.detach())
        return {name: (m.weight.detach().float(), m.bias.detach().float()) for name, m in self.named_modules() if name in REF_LAYERS}

    def set_fp16(self):
        pass   # parameters are created in their final dtype
