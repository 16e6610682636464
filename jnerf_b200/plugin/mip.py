"""MipNerfMLP / MipSampler / Blender: mirror of the reference's contrib/mipnerf (models/networks/mip_network.py:124-222,
models/samplers/mip_sampler/mip_sampler.py, dataset/nerf_datasets.py:22-235) on csrc/mip_sampler.cu and csrc/mip_mlp.cu.  DESIGN.md
section 11.

With using_fp16=True MipNerfMLP is ONE flat fp16 vector in the layout of the vanilla NeRF kernels (plugin/nerf.py), whose forward computes
the integrated positional encoding on chip (ops.mip_fwd) and whose backward is ops.nerf_bwd.  With using_fp16=False (mip_base.py) it is an
fp32 torch.nn.Linear chain under the reference's module names, fed by the fp32 encoder kernel (ops.mip_encode).

Flat layout: the kernel layers of plugin/nerf.py, with the reference's names and column orders mapped as
    layers.0.0       (256, 48)  -> columns 0..47 of kernel layer 0
    layers.5.0       (256, 304) reads [h4, enc]: reference columns 0..255 -> kernel 64..319, 256..303 -> kernel 0..47
    density_layer    (1, 256)   -> row 0 of kernel layer 8;  extra_layer (256, 256) -> rows 16..271
    view_layers.0.0  (128, 283) reads [bottleneck, pos_enc(viewdir)] = [x, sin(2^k x) k<4, cos(2^k x) k<4]; the kernel's view groups hold
                     FrequencyEncoder(4)'s [x, sin(x), cos(x), sin(2x), ...] order, so the 24 sinusoid columns are permuted
    color_layer      (3, 128)   -> rows 0..2 of kernel layer 10"""
import json
import math
import os

import numpy as np
import torch

from .. import ops
from ..utils.config import get_cfg
from ..utils.registry import DATASETS, NETWORKS, SAMPLERS
from . import nerf
from .dataset import SyntheticNerfDataset, fov_to_focal_length
from .module import Module

N_SAMPLES_MAX = 128

_VIEW_COLS = [(0, 0, 256), (256, 256, 3)]
for _k in range(4):
    _VIEW_COLS += [(259 + 3 * _k, 259 + 6 * _k, 3), (271 + 3 * _k, 262 + 6 * _k, 3)]
REF_LAYERS = {f"layers.{i}.0": ((256, 256), i, 0, [(0, 0, 256)]) for i in (1, 2, 3, 4, 6, 7)}
REF_LAYERS.update({
    "layers.0.0": ((256, 48), 0, 0, [(0, 0, 48)]),
    "layers.5.0": ((256, 304), 5, 0, [(0, 64, 256), (256, 0, 48)]),
    "density_layer": ((1, 256), 8, 0, [(0, 0, 256)]),
    "extra_layer": ((256, 256), 8, 16, [(0, 0, 256)]),
    "view_layers.0.0": ((128, 283), 9, 0, _VIEW_COLS),
    "color_layer": ((3, 128), 10, 0, [(0, 0, 128)]),
})
# construction order of the reference's modules (mip_network.py:140-173)
REF_ORDER = [f"layers.{i}.0" for i in range(8)] + ["density_layer", "extra_layer", "view_layers.0.0", "color_layer"]


def pack(ref):
    return nerf.pack(ref, REF_LAYERS)


def unpack(flat):
    return nerf.unpack(flat, REF_LAYERS)


def _encoder_args(cfg):
    return dict(ray_shape=cfg.ray_shape, integrate=not cfg.disable_integration, min_deg=int(cfg.min_deg_point))


@NETWORKS.register_module()
class MipNerfMLP(Module):
    """mip_network.py:124-216 for its only configuration (mip_base.py): depth 8, width 256, skip 4, one 128-wide view layer, degrees
    [min_deg_point, min_deg_point + 8) and deg_view 4.  execute(enc (N, 48), view (N, 27)) -> (N, 4) {raw rgb, raw density}."""

    def __init__(self):
        super().__init__()
        cfg = get_cfg()
        shape = (cfg.net_depth, cfg.net_width, cfg.skip_layer, cfg.net_depth_condition, cfg.net_width_condition, cfg.num_density_channels,
                 cfg.num_rgb_channels, cfg.max_deg_point - cfg.min_deg_point, cfg.deg_view, bool(cfg.use_viewdirs))
        if shape != (8, 256, 4, 1, 128, 1, 3, 8, 4, True):
            raise NotImplementedError("MipNerfMLP: the kernels are built for mip_base.py's network: net_depth 8, net_width 256, skip_layer 4, "
                                      "net_depth_condition 1, net_width_condition 128, 1 density and 3 rgb channels, max_deg_point - "
                                      "min_deg_point = 8, deg_view 4, use_viewdirs")
        self.using_fp16 = bool(cfg.using_fp16)
        self.enc_args = _encoder_args(cfg)
        gen = torch.Generator(device="cuda").manual_seed(int(cfg.seed or 1) + 1)
        ref = nerf.init_reference_params(gen, REF_LAYERS, REF_ORDER)
        if self.using_fp16:
            self.params = torch.nn.Parameter(pack(ref))
            return

        def linear(name):
            (o, i) = REF_LAYERS[name][0]
            lin = torch.nn.Linear(i, o).cuda()
            with torch.no_grad():
                lin.weight.copy_(ref[name][0])
                lin.bias.copy_(ref[name][1])
            return lin
        self.layers = torch.nn.ModuleList([torch.nn.Sequential(linear(f"layers.{i}.0"), torch.nn.ReLU()) for i in range(8)])
        self.density_layer = linear("density_layer")
        self.extra_layer = linear("extra_layer")
        self.view_layers = torch.nn.Sequential(torch.nn.Sequential(linear("view_layers.0.0"), torch.nn.ReLU()))
        self.color_layer = linear("color_layer")

    def execute(self, x, condition):
        """The fp32 chain (mip_network.py:186-216) on per-row encodings."""
        inputs = x
        for i, layer in enumerate(self.layers):
            x = layer(x)
            if i % 4 == 0 and i > 0:
                x = torch.cat([x, inputs], -1)
        raw_density = self.density_layer(x)
        x = self.view_layers(torch.cat([self.extra_layer(x), condition], -1))
        return torch.cat([self.color_layer(x), raw_density], -1)

    def raw(self, rays, t, out=None, saved=None):
        """(R * S, 4) raw outputs of the intervals of t (R, S + 1) along rays (R, 12).  fp16 kernels: out / saved as ops.mip_fwd."""
        if self.using_fp16:
            return ops.mip_fwd(rays, t, self.params, out=out, saved=saved, **self.enc_args)
        enc, view = ops.mip_encode(rays, t, **self.enc_args)
        return self.execute(enc, view)

    def reference_params(self):
        """{reference name: (weight, bias)} in fp32, e.g. layers.5.0 -> ((256, 304), (256,))."""
        if self.using_fp16:
            return unpack(self.params.detach())
        return {name[:-len(".weight")]: (p.detach().float(), self.get_parameter(name[:-len("weight")] + "bias").detach().float())
                for name, p in self.named_parameters() if name.endswith(".weight")}

    def set_fp16(self):
        pass   # parameters are created in their final dtype


@SAMPLERS.register_module()
class MipSampler:
    """mip_sampler.py:11-96.  sample(rays, 0) gives the stratified fenceposts, sample(rays, 1, t, weights) the resampled ones; each call
    with `randomized` takes R (S + 1) draws of the sampler's pcg32 stream (ops.mip_sample / ops.mip_resample) and moves it on past them."""

    def __init__(self, update_den_freq=16):
        cfg = get_cfg()
        if cfg.density_noise and cfg.density_noise > 0:
            raise NotImplementedError("MipSampler: density_noise > 0 is not supported (mip_base.py uses 0)")
        if not 1 <= int(cfg.num_samples) <= N_SAMPLES_MAX:
            raise NotImplementedError(f"MipSampler: num_samples must be in [1, {N_SAMPLES_MAX}] (one warp a ray), got {cfg.num_samples}")
        if cfg.ray_shape not in ops.RAY_SHAPES:
            raise ValueError(f"MipSampler: ray_shape must be one of {ops.RAY_SHAPES}, got {cfg.ray_shape!r}")
        self.num_samples, self.randomized, self.lindisp = int(cfg.num_samples), bool(cfg.randomized), bool(cfg.lindisp)
        self.resample_padding, self.white_bkgd = float(cfg.resample_padding), bool(cfg.white_bkgd)
        self.rgb_padding, self.density_bias = float(cfg.rgb_padding), float(cfg.density_bias)
        self.rng = ops.pcg32_seed(1337 + int(cfg.seed or 0))

    def sample(self, rays, i_level, t_vals=None, weights=None):
        if i_level == 0:
            t = ops.mip_sample(rays, self.num_samples, self.lindisp, self.randomized, self.rng)
        else:
            t = ops.mip_resample(t_vals, weights, self.resample_padding, self.randomized, self.rng)
        if self.randomized:
            ops.pcg32_advance(self.rng, rays.shape[0] * (self.num_samples + 1))
        return t

    def rays2rgb(self, rays, raw, t_vals, weights=True):
        """(rgb, acc, distance, weights or None) of raw network outputs for the intervals of t_vals."""
        return ops.mip_composite_fwd(raw, t_vals, rays, self.rgb_padding, self.density_bias, self.white_bkgd, weights)

    def state_dict(self):
        return {"rng": torch.from_numpy(self.rng.astype(np.int64))}

    def load_state_dict(self, sd):
        self.rng[:] = sd["rng"].cpu().numpy().astype(np.uint64)


class _BlenderRays:
    """The device half of Blender: shuffled pixel ids of all training images, and rays + targets made per batch (ops.mip_rays).
    Needs n_images, H, W, focal, c2w ((n, 12) row-major 3x4, NeRF camera-to-world), image_data ((n * H * W, 4) uint8), near, far."""

    def _finish_init(self, seed):
        self.resolution = [self.W, self.H]
        self.n_examples = self.n_images
        self.idx_now = 0
        self._gen = torch.Generator(device="cuda").manual_seed(int(seed))
        self.shuffle_index = torch.randperm(self.n_images * self.H * self.W, device="cuda", generator=self._gen).int()

    def rays_for(self, pix):
        return ops.mip_rays(pix.contiguous(), self.W, self.H, self.c2w, self.focal, self.near, self.far, self.image_data)

    def __next__(self):
        """nerf_datasets.py:52-63: the next batch_size pixels of the shuffled list (reshuffled when it runs out) -> (rays, target)."""
        n = self.n_images * self.H * self.W
        if self.idx_now + self.batch_size >= n:
            self.shuffle_index = torch.randperm(n, device="cuda", generator=self._gen).int()
            self.idx_now = 0
        pix = self.shuffle_index[self.idx_now:self.idx_now + self.batch_size]
        self.idx_now += self.batch_size
        return self.rays_for(pix)

    def image_rays(self, img_id):
        """(rays (H * W, 12), target (H * W, 3)) of image img_id in row-major pixel order."""
        pix = torch.arange(self.H * self.W, device="cuda", dtype=torch.int32) + int(img_id) * self.H * self.W
        return self.rays_for(pix)


@DATASETS.register_module()
class Blender(_BlenderRays):
    """nerf_datasets.py:22-150: NeRF-synthetic transforms_{mode}.json (train also takes the val files; val and test take frames[::10]),
    frames without an image on disk skipped, the focal length from fl_x or camera_angle_x, uint8 RGBA images."""

    def __init__(self, root_dir, batch_size, mode="train", H=0, W=0, near=0., far=1., img_alpha=True, have_img=True, preload_shuffle=True, seed=0):
        from PIL import Image
        assert mode in ("train", "val", "test")
        if not have_img:
            raise NotImplementedError("Blender: have_img=False (rays without images) is not supported")
        self.root_dir, self.batch_size, self.mode, self.H, self.W = root_dir, batch_size, mode, H, W
        self.near, self.far = float(near), float(far)
        json_data = None
        for root, _, files in sorted(os.walk(root_dir)):
            for f in sorted(files):
                stem, ext = os.path.splitext(f)
                if ext == ".json" and (mode in stem or (mode == "train" and "val" in stem)):
                    with open(os.path.join(root, f)) as fh:
                        d = json.load(fh)
                    if json_data is None:
                        json_data = d
                    else:
                        json_data["frames"] += d["frames"]
        if json_data is None:
            raise FileNotFoundError(f"Blender: no transforms json for mode {mode!r} under {root_dir}")
        frames = json_data["frames"][::10] if mode in ("val", "test") else json_data["frames"]
        imgs, mats = [], []
        for fr in frames:
            p = os.path.join(root_dir, fr["file_path"][2:])
            if not os.path.exists(p):
                p += ".png"
                if not os.path.exists(p):
                    continue
            im = np.asarray(Image.open(p))
            if im.ndim == 2:
                im = im[..., None].repeat(3, -1)
            if im.shape[-1] == 3:
                im = np.concatenate([im, np.full(im.shape[:2] + (1,), 255, np.uint8)], -1)
            if self.H == 0 or self.W == 0:
                self.H, self.W = im.shape[0], im.shape[1]
            imgs.append(im)
            mats.append(np.array(fr["transform_matrix"], np.float32)[:3, :4])
        self.n_images = len(imgs)
        if "fl_x" in json_data:
            self.focal = float(json_data["fl_x"])
        elif "camera_angle_x" in json_data:
            self.focal = fov_to_focal_length(self.W, json_data["camera_angle_x"] * 180 / math.pi)
        else:
            self.focal = 0.0
        self.c2w = torch.from_numpy(np.stack(mats).reshape(-1, 12)).to("cuda")
        self.image_data = torch.from_numpy(np.stack(imgs).reshape(-1, 4)).to("cuda")
        self._finish_init(seed)


@DATASETS.register_module()
class SyntheticBlender(_BlenderRays):
    """Blender on the procedural stand-in of the lego scene: SyntheticNerfDataset's cameras (NeRF camera-to-world) and images."""

    def __init__(self, batch_size, mode="train", near=0., far=1., n_images=100, H=800, W=800, seed=0, root_dir=None, preload_shuffle=True):
        ds = SyntheticNerfDataset(batch_size=batch_size, mode=mode, n_images=n_images, H=H, W=W, seed=seed)
        self.batch_size, self.mode, self.H, self.W, self.n_images = batch_size, mode, ds.H, ds.W, ds.n_images
        self.near, self.far, self.focal = float(near), float(far), float(ds._focal[0])
        self.c2w = torch.from_numpy(np.stack([p[:3, :4] for p in ds.poses]).reshape(-1, 12)).to("cuda")
        self.image_data = ds.image_data.reshape(-1, 4)
        self._finish_init(seed)


@DATASETS.register_module()
class Blenders:
    """nerf_datasets.py's multi-camera (multiscale) dataset of multicam.py: not supported."""

    def __init__(self, *a, **k):
        raise NotImplementedError("Blenders (the multiscale multicam dataset) is not supported; use Blender")
