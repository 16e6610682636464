"""pixelNeRF (the reference's contrib/pixelnerf): parameters under the reference's names, the flat fp16 layout of csrc/pixelnerf.cu, the
frozen image encoder, the reference views and the tiny_nerf_data.npz loader.  DESIGN.md section 13."""
import math
import warnings

import numpy as np
import torch

WIDTH, ENC_COLS, ENC_PAD, N_F1, N_F2 = 512, 42, 64, 3, 2


def _linears():
    """(name, out, in, padded in) of every Linear, in the flat layout's order (Network.py:46-64)."""
    out = [("mlp.0", WIDTH, ENC_COLS, ENC_PAD)]
    for i in range(N_F1):
        out += [(f"f1.{i}.img_mlp.0", WIDTH, WIDTH, WIDTH), (f"f1.{i}.mlp.0", WIDTH, WIDTH, WIDTH), (f"f1.{i}.mlp.2", WIDTH, WIDTH, WIDTH)]
    for i in range(N_F2):
        out += [(f"f2.{i}.mlp.0", WIDTH, WIDTH, WIDTH), (f"f2.{i}.mlp.2", WIDTH, WIDTH, WIDTH)]
    return out + [("final_layer", 4, WIDTH, WIDTH)]


LINEARS = _linears()
N_PARAMS = sum(o * i + o for _, o, i, _ in LINEARS)                  # 3 438 596, the reference's count
N_FLAT = sum(o * p + o for _, o, _, p in LINEARS)                    # the flat layout: mlp.0 padded to 64 input columns


def flat_offsets():
    """name -> (weight offset, bias offset) into the flat vector."""
    off, out = 0, {}
    for name, o, _, p in LINEARS:
        out[name] = (off, off + o * p)
        off += o * p + o
    return out


def pack(state, dtype=torch.float32):
    """A state dict under the reference's names -> the flat vector (pad columns zero)."""
    offs = flat_offsets()
    dev = next(iter(state.values())).device
    flat = torch.zeros(N_FLAT, dtype=dtype, device=dev)
    for name, o, i, p in LINEARS:
        w0, b0 = offs[name]
        flat[w0:b0].view(o, p)[:, :i] = state[f"{name}.weight"].to(dtype)
        flat[b0:b0 + o] = state[f"{name}.bias"].to(dtype)
    return flat


def unpack(flat):
    """The flat vector -> a state dict of fp32 tensors under the reference's names."""
    offs = flat_offsets()
    out = {}
    for name, o, i, p in LINEARS:
        w0, b0 = offs[name]
        out[f"{name}.weight"] = flat[w0:b0].view(o, p)[:, :i].float().clone()
        out[f"{name}.bias"] = flat[b0:b0 + o].float().clone()
    return out


def init_state(seed=0):
    """torch's default nn.Linear initialisation of every layer, seeded, on the CPU."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, o, i, _ in LINEARS:
        bound = 1.0 / math.sqrt(i)                         # kaiming_uniform(a=sqrt(5)) and the bias rule both give U(-1/sqrt(in), 1/sqrt(in))
        out[f"{name}.weight"] = (torch.rand((o, i), generator=g) * 2 - 1) * bound
        out[f"{name}.bias"] = (torch.rand(o, generator=g) * 2 - 1) * bound
    return out


class PixelNeRF(torch.nn.Module):
    """The network of Network.py as the kernels read it: `params` (flat fp16), the fp32 master copy and Adam's moments."""

    def __init__(self, state=None, seed=0, device="cuda"):
        super().__init__()
        state = init_state(seed) if state is None else state
        master = pack({k: v.to(device) for k, v in state.items()})
        self.register_buffer("master", master)
        self.register_buffer("params", master.half())
        self.register_buffer("m", torch.zeros_like(master))
        self.register_buffer("v", torch.zeros_like(master))

    def reference_state(self):
        return unpack(self.master)

    def load_reference_state(self, state):
        self.master.copy_(pack({k: v.to(self.master.device) for k, v in state.items()}))
        self.params.copy_(self.master.half())
        self.m.zero_()
        self.v.zero_()


# ---- the fp32 torch restatement of Network.py + Dataset.py:86-94 (the parity reference and the cuBLAS comparison) ----------------------
def positional_encoding(x, d):
    """Network.py:5-11 + :73-77: [x, sin(2^i 1.5 x), cos(2^i 1.5 x) for i < 6, d / |d|] (..., 42)."""
    pe = [x]
    for i in range(6):
        pe += [torch.sin(2.0 ** i * x * 1.5), torch.cos(2.0 ** i * x * 1.5)]
    dn = d / d.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    return torch.cat(pe + [dn.expand_as(x)], -1)


def project(pts, cams, scale, pixel_aligned=False):
    """Dataset.py:86-93: uv (n_ref, ...pts, 2) of pts (..., 3) in each reference (cams (n_ref, 12))."""
    Rt, pos = cams[:, :9].reshape(-1, 3, 3), cams[:, 9:]
    shp = pts.shape[:-1]
    p = torch.einsum("kij,knj->kni", Rt, pts.reshape(1, -1, 3) - pos[:, None])
    uv = p[..., :2] / p[..., 2:] / scale
    uv = -uv if pixel_aligned else uv
    uv = torch.stack([uv[..., 0], -uv[..., 1]], -1)
    return uv.reshape((cams.shape[0],) + shp + (2,))


def feature_matching(feats, pts, cams, scale, pixel_aligned=False):
    """grid_sample(align_corners=True, padding_mode="border") of the (n_ref, fh, fw, C) maps at pts (N, 3) -> (n_ref, N, C)."""
    uv = project(pts, cams, scale, pixel_aligned).to(feats.dtype)
    f = torch.nn.functional.grid_sample(feats.permute(0, 3, 1, 2), uv[:, :, None, :], align_corners=True, padding_mode="border")
    return f[..., 0].permute(0, 2, 1)


def network_torch(state, enc, feat, dtype=torch.float32):
    """Network.py:66-94 on enc (N, 42) and feat (n_ref, N, 512): raw (N, 4) = (relu(o0), sigmoid(o1:4)).  The stem runs once per sample."""
    lin = lambda name, x: torch.nn.functional.linear(x, state[f"{name}.weight"].to(dtype), state[f"{name}.bias"].to(dtype))
    relu = torch.relu
    f = relu(lin("mlp.0", enc.to(dtype)))[None].expand(feat.shape[0], -1, -1)
    feat = feat.to(dtype)
    for i in range(N_F1):
        x = f + relu(lin(f"f1.{i}.img_mlp.0", feat))
        f = relu(lin(f"f1.{i}.mlp.2", relu(lin(f"f1.{i}.mlp.0", x)))) + x
    f = f.mean(0)
    for i in range(N_F2):
        f = relu(lin(f"f2.{i}.mlp.2", relu(lin(f"f2.{i}.mlp.0", f)))) + f
    o = lin("final_layer", f)
    return torch.cat([relu(o[:, :1]), torch.sigmoid(o[:, 1:])], -1)


def composite_torch(raw, z, rays):
    """Render.py:16-18 + :34-46: (rgb (R, 3), depth (R,), acc (R,)) of raw (R S, 4) = (sigma, c)."""
    R, S = rays.shape[0], z.shape[0]
    raw = raw.reshape(R, S, 4)
    delta = torch.cat([z[1:] - z[:-1], z.new_full((1,), 1e10)])[None] * rays[:, 3:6].norm(dim=-1, keepdim=True)
    alpha = 1 - torch.exp(-raw[..., 0] * delta)
    T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-7], -1), -1)[:, :-1]
    w = alpha * T
    return (w[..., None] * raw[..., 1:]).sum(1), (w * z).sum(-1), w.sum(-1)


# ---- rays, encoder, reference views, data ----------------------------------------------------------------------------------------------
def sample_rays_np(H, W, f, c2w):
    """Dataset.py:8-13."""
    i, j = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing="xy")
    dirs = np.stack([(i - W * .5 + 0.5) / f, -(j - H * .5 + 0.5) / f, -np.ones_like(i)], -1)
    rays_d = np.sum(dirs[..., None, :] * c2w[:3, :3], -1)
    rays_o = np.broadcast_to(c2w[:3, -1], np.shape(rays_d))
    return rays_o, rays_d


class ImageEncoder(torch.nn.Module):
    """ImageEncoder.py: resnet34 conv1 / bn1 / relu, layer1 (after maxpool), layer2, layer3, each resized bilinearly (align_corners) to the
    conv1 size and concatenated: 64 + 64 + 128 + 256 = 512 channels at H/2 x W/2.  Frozen, eval mode.  weights: a torchvision-layout resnet34
    state dict (the reference loads ImageNet weights, which cannot be downloaded here); None: seeded He initialisation, with a warning."""

    def __init__(self, weights=None, seed=0):
        super().__init__()
        import torchvision
        with torch.random.fork_rng(devices=[]):                    # seeds the initialisation without touching the caller's RNG
            torch.manual_seed(seed)
            self.resnet = torchvision.models.resnet34(weights=None)
        if weights is None:
            warnings.warn("pixelNeRF ImageEncoder: no encoder_weights given, using a seeded He-initialised resnet34 (not the reference's "
                          "ImageNet weights)")
        else:
            # the encoder never reads the classifier (fc); every other resnet34 tensor must be present and nothing else may be
            missing, unexpected = self.resnet.load_state_dict(weights, strict=False)
            bad = [k for k in missing if not k.startswith("fc.") and not k.endswith("num_batches_tracked")] + list(unexpected)
            if bad:
                raise ValueError(f"pixelNeRF ImageEncoder: encoder_weights is not a torchvision resnet34 state dict: missing / unexpected "
                                 f"keys {bad[:8]}{' ...' if len(bad) > 8 else ''}")
        self.eval()

    @torch.no_grad()
    def forward(self, x):
        r = self.resnet
        f1 = r.relu(r.bn1(r.conv1(x)))
        f2 = r.layer1(r.maxpool(f1))
        f3 = r.layer2(f2)
        f4 = r.layer3(f3)
        sz = f1.shape[-2:]
        lat = [torch.nn.functional.interpolate(f, sz, mode="bilinear", align_corners=True) for f in (f1, f2, f3, f4)]
        return torch.cat(lat, 1)


def pack_cams(c2w):
    """(n_ref, 12) fp32: R_t = c2w[:3,:3]^T row-major, then the camera position (Dataset.py:79-80)."""
    c2w = torch.as_tensor(np.asarray(c2w, np.float32))
    return torch.cat([c2w[:, :3, :3].transpose(1, 2).reshape(-1, 9), c2w[:, :3, 3]], 1).contiguous()


class ReferenceViews:
    """Dataset.py:74-94: the reference views' feature maps (n_ref, H/2, W/2, 512) fp16 channel-last, the packed cameras and scale."""

    def __init__(self, images, c2w, focal, encoder=None, device="cuda", pixel_aligned=False):
        images = torch.as_tensor(np.asarray(images, np.float32)).to(device)
        encoder = ImageEncoder() if encoder is None else encoder
        feats = encoder.to(images.device)(images.permute(0, 3, 1, 2))
        self.feats = feats.permute(0, 2, 3, 1).contiguous().half()
        self.cams = pack_cams(c2w).to(device)
        self.c2w = np.asarray(c2w, np.float32)
        self.H = images.shape[1]
        self.focal = float(focal)
        self.scale = (self.H / 2) / self.focal
        self.pixel_aligned = bool(pixel_aligned)


class TinyNerfData:
    """tiny_nerf_data.npz (images (N, H, W, 3) fp32, poses (N, 4, 4), focal): the first n_train views are the reference views and the
    training images (main.py:12-16); the rest are held out.  Rays (n_train H W, 9) = o, d, rgb (Dataset.py:43-59), on the device."""

    def __init__(self, path, n_train=3, device="cuda"):
        d = np.load(path)
        self.images, self.poses, self.focal = d["images"].astype(np.float32), d["poses"].astype(np.float32), float(d["focal"])
        self.n_train = int(n_train)
        self.H, self.W = self.images.shape[1:3]
        rows = []
        for i in range(self.n_train):
            o, dd = sample_rays_np(self.H, self.W, self.focal, self.poses[i])
            rows.append(np.concatenate([o.reshape(-1, 3), dd.reshape(-1, 3), self.images[i].reshape(-1, 3)], 1))
        self.rays = torch.from_numpy(np.concatenate(rows, 0)).to(device)
        self.device = device

    def batches(self, batch_size, generator):
        """One epoch: the rays shuffled on the device, in batches of batch_size, drop_last (main.py:20)."""
        perm = torch.randperm(self.rays.shape[0], generator=generator, device=self.rays.device)
        for k in range(self.rays.shape[0] // batch_size):
            yield self.rays[perm[k * batch_size:(k + 1) * batch_size]]

    def image_rays(self, c2w):
        """(H W, 6) rays of a camera."""
        o, d = sample_rays_np(self.H, self.W, self.focal, np.asarray(c2w, np.float32))
        return torch.from_numpy(np.concatenate([o.reshape(-1, 3), d.reshape(-1, 3)], 1).astype(np.float32)).to(self.device)
