"""NerfDataset (mirror of dataset/dataset.py:16-270) and SyntheticNerfDataset, the stand-in used when the
NeRF-synthetic `lego` scene is unavailable (the reference downloads it at run time, dataset_util.py:101-109).

Both expose what the sampler / runner read: n_images, resolution [W,H], aabb_scale, aabb_range, metadata (n,11),
focal_lengths (n,2), transforms_gpu (n, 3x4 stored column-major = 12 floats, dataset.py:164-165), image_data
(n, H*W, 4), batch_size and __next__() -> (img_ids, rays_o, rays_d, rgba)."""
import json
import math
import os

import numpy as np
import torch

from .. import ops
from ..utils.registry import DATASETS

NERF_SCALE = 0.33
DEVICE = "cuda"          # where the image / pose tensors live; tests of the file parsing set this to "cpu"


def fov_to_focal_length(resolution, degrees):
    return 0.5 * resolution / math.tan(0.5 * degrees * math.pi / 180)


def matrix_nerf2ngp(matrix, scale, offset, correct_pose=(1, -1, -1)):
    """dataset.py:255-262: 3x4 camera-to-world, NeRF -> NGP convention (axis cycle, scale 0.33, offset 0.5)."""
    m = np.array(matrix, np.float32)[:3, :].copy()
    m[:, 0] *= correct_pose[0]
    m[:, 1] *= correct_pose[1]
    m[:, 2] *= correct_pose[2]
    m[:, 3] = m[:, 3] * scale + np.asarray(offset, np.float32)
    return m[[1, 2, 0]]


class _RayBatcher:
    """Pixel shuffling + device ray generation shared by both datasets (dataset.py:57-66,172-188)."""

    def _finish_init(self):
        dev = DEVICE
        self.resolution = [self.W, self.H]
        self.n_images = len(self._xforms)
        xf = np.stack(self._xforms).astype(np.float32)                       # (n,3,4)
        self.transforms_gpu = torch.from_numpy(np.ascontiguousarray(xf.transpose(0, 2, 1)).reshape(self.n_images, 12)).to(dev)
        self.focal_lengths = torch.tensor([self._focal] * self.n_images, dtype=torch.float32, device=dev)
        md = np.zeros((self.n_images, 11), np.float32)
        md[:, 4], md[:, 5] = self._cx / self.W, self._cy / self.H
        md[:, 6], md[:, 7] = self._focal
        self.metadata = torch.from_numpy(md).to(dev)
        self.principal = self.metadata[:, 4:6].contiguous()
        self.aabb_range = (0.5 - self.aabb_scale / 2, 0.5 + self.aabb_scale / 2)    # dataset.py:155-156
        self.idx_now = 0
        self._gen = torch.Generator(device=dev).manual_seed(int(self.seed))
        self.shuffle_index = torch.randperm(self.n_images * self.H * self.W, device=dev, generator=self._gen).int()

    def next_pixels(self, n=None):
        """The next n entries of the shuffled pixel list; the list is reshuffled in place when it runs out."""
        n = self.batch_size if n is None else n
        if self.idx_now + n >= self.shuffle_index.shape[0]:
            self.shuffle_index.copy_(torch.randperm(self.n_images * self.H * self.W, device=DEVICE, generator=self._gen).int())
            self.idx_now = 0
        start = self.idx_now
        self.idx_now += n
        return self.shuffle_index[start:start + n]

    def rays_for(self, pix):
        return ops.raygen(pix.contiguous(), self.W, self.H, self.transforms_gpu, self.focal_lengths, self.principal)

    def rgba_for(self, pix):
        v = self.image_data.reshape(-1, 4)[pix.long()]
        return v.float() / 255.0 if v.dtype == torch.uint8 else v

    def __next__(self):
        pix = self.next_pixels()
        img_ids, rays_o, rays_d = self.rays_for(pix)
        return img_ids, rays_o, rays_d, self.rgba_for(pix)

    def generate_rays_total_test(self, img_id):
        """All rays of one image in row-major pixel order (dataset.py:214-238)."""
        pix = torch.arange(self.H * self.W, device=DEVICE, dtype=torch.int32) + int(img_id) * self.H * self.W
        _, o, d = self.rays_for(pix)
        return o, d


@DATASETS.register_module()
class NerfDataset(_RayBatcher):
    def __init__(self, root_dir, batch_size, mode="train", H=0, W=0, correct_pose=(1, -1, -1), aabb_scale=None, scale=None, offset=None,
                 img_alpha=True, to_jt=True, have_img=True, preload_shuffle=True, seed=0):
        from PIL import Image
        assert mode in ("train", "val", "test")
        self.root_dir, self.batch_size, self.mode, self.seed = root_dir, batch_size, mode, seed
        self.scale = NERF_SCALE if scale is None else scale
        self.offset = [0.5, 0.5, 0.5] if offset is None else offset
        json_data = None
        for root, _, files in os.walk(root_dir):
            for f in sorted(files):
                stem, ext = os.path.splitext(f)
                if ext == ".json" and (mode in stem or (mode == "train" and "val" in stem)):      # dataset.py:77
                    with open(os.path.join(root, f)) as fh:
                        d = json.load(fh)
                    if json_data is None:
                        json_data = d
                    else:
                        json_data["frames"] += d["frames"]
        assert json_data is not None, f"dataset is not found at {root_dir}"
        self.H, self.W = int(json_data.get("h", H)), int(json_data.get("w", W))
        frames = json_data["frames"][::10] if mode == "val" else json_data["frames"]
        imgs, self._xforms, self.poses = [], [], []
        self.correct_pose = tuple(correct_pose)
        for fr in frames:
            p = os.path.join(root_dir, fr["file_path"])
            if not os.path.exists(p):
                p += ".png"
                if not os.path.exists(p):
                    continue                                                                        # dataset.py:103-107
            im = np.asarray(Image.open(p))
            if im.ndim == 2:
                im = im[..., None].repeat(3, -1)
            if im.shape[-1] == 3:
                im = np.concatenate([im, np.full(im.shape[:2] + (1,), 255, np.uint8)], -1)
            if self.H == 0 or self.W == 0:
                self.H, self.W = im.shape[0], im.shape[1]
            imgs.append(im)
            self.poses.append(np.array(fr["transform_matrix"], np.float32))                           # NeRF camera-to-world, as in the file
            self._xforms.append(matrix_nerf2ngp(fr["transform_matrix"], self.scale, self.offset, correct_pose))
        self.image_data = torch.from_numpy(np.stack(imgs)).to(DEVICE).reshape(len(imgs), -1, 4)
        def read_focal_length(resolution, axis):                                                   # dataset.py:125-131
            if "fl_" + axis in json_data:
                return float(json_data["fl_" + axis])
            if "camera_angle_" + axis in json_data:
                return fov_to_focal_length(resolution, json_data["camera_angle_" + axis] * 180 / math.pi)
            return 0.0
        x_fl, y_fl = read_focal_length(self.W, "x"), read_focal_length(self.H, "y")
        if x_fl != 0:                                                                               # :134-142
            self._focal = (x_fl, y_fl if y_fl != 0 else x_fl)
        elif y_fl != 0:
            self._focal = (y_fl, y_fl)
        else:
            raise RuntimeError("Couldn't read fov.")
        self._cx, self._cy = json_data.get("cx", self.W / 2), json_data.get("cy", self.H / 2)
        self.aabb_scale = json_data.get("aabb_scale", 1) if aabb_scale is None else aabb_scale
        self.have_img = have_img
        self._finish_init()


def synthetic_cameras(n_images, radius=4.0, seed=0, azimuth=(0.0, 360.0), elevation=(5.0, 85.0)):
    """Camera-to-world matrices (NeRF/blender convention, looking at the origin) on a sphere of `radius`,
    upper hemisphere like NeRF-synthetic (cf. dataset/camera_path.py:27-28 which also uses radius 4); `azimuth` / `elevation`
    (degrees) restrict the cap, e.g. to the frontal arc of a hand-held capture like data/fox."""
    rng = np.random.default_rng(seed)
    mats = []
    for _ in range(n_images):
        theta = rng.uniform(math.radians(azimuth[0]), math.radians(azimuth[1]))
        phi = rng.uniform(math.radians(elevation[0]), math.radians(elevation[1]))
        pos = radius * np.array([math.cos(theta) * math.cos(phi), math.sin(theta) * math.cos(phi), math.sin(phi)])
        fwd = -pos / np.linalg.norm(pos)                 # camera looks along -z
        right = np.cross(fwd, np.array([0, 0, 1.0]))
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        m = np.eye(4)
        m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, up, -fwd, pos
        mats.append(m)
    return mats


@DATASETS.register_module()
class SyntheticNerfDataset(_RayBatcher):
    """Procedural stand-in for NeRF-synthetic lego: `n_images` 800x800 RGBA views (camera_angle_x 0.6911, radius 4,
    aabb_scale 1) of an analytic scene -- a few shaded, textured spheres on a slab -- ray-traced on the GPU at start-up."""

    SPHERES = [  # centre (NeRF world units), radius, base colour
        ((0.0, 0.0, 0.1), 0.55, (0.85, 0.25, 0.2)),
        ((0.7, 0.2, -0.1), 0.3, (0.2, 0.6, 0.85)),
        ((-0.5, 0.6, 0.25), 0.25, (0.95, 0.8, 0.2)),
        ((-0.3, -0.7, -0.15), 0.35, (0.3, 0.8, 0.35)),
        ((0.35, -0.55, 0.45), 0.2, (0.8, 0.4, 0.85)),
    ]
    SLAB_Z, SLAB_HALF, SLAB_THICK = -0.5, 1.0, 0.08
    # style "fox": stand-in for the reference's data/fox (BASELINE config #3) with that capture's numbers
    # (data/fox/transforms_train.json: 1080x1920 portrait frames, fl 1375.52 / 1374.49, principal point (554.558, 965.268),
    # aabb_scale 4, 50 frames on disk, cameras ~5.15 NeRF units from the subject in a frontal arc, opaque RGB images):
    # the same analytic objects enlarged so that they leave the unit cube (cascades 1 and 2 of the occupancy grid fill up),
    # seen from inside an opaque textured backdrop sphere -- every pixel has alpha 1, as in a JPEG capture.
    FOX = dict(H=1920, W=1080, fl=(1375.52, 1374.49), c=(554.558, 965.268), aabb_scale=4, n_images=50, radius=5.15, azimuth=(-55.0, 55.0),
               elevation=(-8.0, 30.0), obj_scale=2.2, backdrop_radius=1.9)

    def __init__(self, batch_size=4096, mode="train", n_images=100, H=800, W=800, camera_angle_x=0.6911112070083618, aabb_scale=1, seed=0,
                 root_dir=None, preload_shuffle=True, style="lego"):
        assert style in ("lego", "fox")
        self.batch_size, self.mode, self.seed, self.style = batch_size, mode, seed, style
        self.scale, self.offset = NERF_SCALE, [0.5, 0.5, 0.5]
        self.obj_scale, self.backdrop_radius = 1.0, None
        if style == "fox":
            F = self.FOX
            # explicit H / W (e.g. a reduced test size) keep the capture's aspect, field of view and principal-point offsets
            full = (H, W) in ((800, 800), (0, 0), (F["H"], F["W"]))
            self.H, self.W = (F["H"], F["W"]) if full else (H, W)
            k = self.W / F["W"]
            self._focal = (F["fl"][0] * k, F["fl"][1] * self.H / F["H"])
            self._cx, self._cy = F["c"][0] * k, F["c"][1] * self.H / F["H"]
            self.aabb_scale = F["aabb_scale"]
            self.obj_scale, self.backdrop_radius = F["obj_scale"], F["backdrop_radius"]
            n_images = F["n_images"] if n_images == 100 else n_images
            n = n_images if mode == "train" else max(1, n_images // 10)
            mats = synthetic_cameras(n, radius=F["radius"], seed=seed + (0 if mode == "train" else 1000), azimuth=F["azimuth"], elevation=F["elevation"])
        else:
            self.H, self.W, self.aabb_scale = H, W, aabb_scale
            n = n_images if mode == "train" else max(1, n_images // 10)
            mats = synthetic_cameras(n, seed=seed + (0 if mode == "train" else 1000))
            fx = fov_to_focal_length(W, camera_angle_x * 180 / math.pi)
            self._focal = (fx, fx)
            self._cx, self._cy = W / 2, H / 2
        self.poses = [np.array(m, np.float32) for m in mats]                                    # NeRF camera-to-world
        self.correct_pose = (1, -1, -1)
        self._xforms = [matrix_nerf2ngp(m, self.scale, self.offset) for m in mats]
        self.have_img = True
        self._finish_init()
        self.image_data = self._render_all()

    # -- analytic renderer (NGP coordinates: world * 0.33 + 0.5, axes cycled like matrix_nerf2ngp) --------------
    def _to_ngp(self, p):
        p = np.asarray(p, np.float32) * self.scale + 0.5
        return p[[1, 2, 0]]

    def _render_all(self):
        out = torch.empty((self.n_images, self.H * self.W, 4), dtype=torch.uint8, device=DEVICE)
        for i in range(self.n_images):
            o, d = self.generate_rays_total_test(i)
            out[i] = (self.shade(o, d) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8)
        return out

    def shade(self, o, d):
        """RGBA in [0,1] of the analytic scene along rays (o,d) given in NGP coordinates."""
        n = o.shape[0]
        t_best = torch.full((n,), float("inf"), device=o.device)
        col = torch.zeros((n, 3), device=o.device)
        nrm = torch.zeros((n, 3), device=o.device)
        light = torch.tensor(self._to_ngp((0.4, -0.3, 1.0)) - 0.5, device=o.device)
        light = light / light.norm()
        k = float(getattr(self, "obj_scale", 1.0))
        for c, r, base in self.SPHERES:
            c_n = torch.tensor(self._to_ngp(tuple(k * x for x in c)), device=o.device)
            r_n = r * self.scale * k
            oc = o - c_n
            b = (oc * d).sum(-1)
            disc = b * b - ((oc * oc).sum(-1) - r_n * r_n)
            t = -b - torch.sqrt(disc.clamp_min(0))
            hit = (disc > 0) & (t > 0) & (t < t_best)
            p = o + t[:, None] * d
            nn_ = (p - c_n) / r_n
            tex = 0.75 + 0.25 * torch.sin(40.0 * p[:, 0]) * torch.sin(40.0 * p[:, 1]) * torch.sin(40.0 * p[:, 2])
            cc = torch.tensor(base, device=o.device)[None, :] * tex[:, None]
            t_best = torch.where(hit, t, t_best)
            col = torch.where(hit[:, None], cc, col)
            nrm = torch.where(hit[:, None], nn_, nrm)
        # slab: axis-aligned box in NeRF world coordinates -> box in NGP coordinates
        lo = torch.tensor(self._to_ngp((-k * self.SLAB_HALF, -k * self.SLAB_HALF, k * (self.SLAB_Z - self.SLAB_THICK))), device=o.device)
        hi = torch.tensor(self._to_ngp((k * self.SLAB_HALF, k * self.SLAB_HALF, k * self.SLAB_Z)), device=o.device)
        lo, hi = torch.minimum(lo, hi), torch.maximum(lo, hi)
        inv = 1.0 / d
        t0, t1 = (lo - o) * inv, (hi - o) * inv
        tn, tf = torch.minimum(t0, t1), torch.maximum(t0, t1)
        tnear, axis = tn.max(-1)
        tfar = tf.min(-1).values
        hit = (tnear < tfar) & (tnear > 0) & (tnear < t_best)
        p = o + tnear[:, None] * d
        chk = ((torch.floor(p[:, 0] * 24) + torch.floor(p[:, 1] * 24) + torch.floor(p[:, 2] * 24)) % 2)
        cc = (0.55 + 0.3 * chk)[:, None] * torch.tensor((0.9, 0.9, 0.85), device=o.device)[None, :]
        bn = torch.zeros_like(nrm)
        bn.scatter_(1, axis[:, None], -torch.sign(d.gather(1, axis[:, None])))
        t_best = torch.where(hit, tnear, t_best)
        col = torch.where(hit[:, None], cc, col)
        nrm = torch.where(hit[:, None], bn, nrm)
        rb = getattr(self, "backdrop_radius", None)
        if rb is not None:
            # opaque backdrop: the inside of a sphere of radius rb (NGP units) around the scene centre, latitude / longitude pattern
            ctr = torch.full((3,), 0.5, device=o.device)
            oc = o - ctr
            b = (oc * d).sum(-1)
            t = -b + torch.sqrt((b * b - ((oc * oc).sum(-1) - rb * rb)).clamp_min(0))
            hit = ~torch.isfinite(t_best) & (t > 0)
            p = o + t[:, None] * d
            q = (p - ctr) / rb
            lon, lat = torch.atan2(q[:, 1], q[:, 0]), torch.asin(q[:, 2].clamp(-1, 1))
            chk = (torch.floor(lon * (12 / math.pi)) + torch.floor(lat * (12 / math.pi))) % 2
            cc = torch.stack([0.35 + 0.25 * chk, 0.45 + 0.2 * torch.sin(3 * lat), 0.6 - 0.2 * chk], -1)
            t_best = torch.where(hit, t, t_best)
            col = torch.where(hit[:, None], cc, col)
            nrm = torch.where(hit[:, None], -q, nrm)
        alpha = torch.isfinite(t_best).float()
        lam = 0.35 + 0.65 * (nrm * light).sum(-1).clamp_min(0)
        rgb = (col * lam[:, None]).clamp(0, 1) * alpha[:, None]
        return torch.cat([rgb, alpha[:, None]], -1)
