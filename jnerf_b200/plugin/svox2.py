"""SparseGrid / SvoxNeRFDataset: mirror of the reference's contrib/plenoxel (models/networks/svox2_network.py, dataset/svox_dataset.py)
on csrc/svox.cu.  DESIGN.md section 12.

The grid is plain device tensors under the reference's names: `_links` (X, Y, Z) int32 (< 0: empty cell), `density_data` (capacity, 1)
and `sh_data` (capacity, 27) fp32, `_offset` / `_scaling` (world -> [0, 1]^3).  Only what the reference's Svox2Runner runs is built: the
SH basis of degree 2, no background model, no NDC or spheric clip, no sigma noise."""
import json
import math
import os
from functools import reduce

import numpy as np
import torch

from .. import ops
from ..utils.registry import DATASETS, NETWORKS

BASIS_TYPE_SH = 1


def gen_morton(D):
    """svox2_utils.py:48-79: the Morton code of every cell of a D^3 grid, (D, D, D) int64 in (x, y, z) order."""
    def expand(v):
        v = (v | (v << 16)) & 0x030000FF
        v = (v | (v << 8)) & 0x0300F00F
        v = (v | (v << 4)) & 0x030C30C3
        return (v | (v << 2)) & 0x09249249
    a = np.arange(D, dtype=np.int64)
    X, Y, Z = np.meshgrid(a, a, a, indexing="ij")
    return (expand(X) << 2) + (expand(Y) << 1) + expand(Z)


class RenderOptions:
    """svox2_utils.py:338-372 defaults: SparseGrid.setup_render_opts is never called by the reference's runner, so these are what runs."""

    def __init__(self):
        self.step_size, self.sigma_thresh, self.stop_thresh, self.background_brightness = 0.5, 1e-10, 1e-7, 1.0
        self.last_sample_opaque, self.near_clip, self.use_spheric_clip = False, 0.0, False

    def as_array(self):
        return (self.step_size, self.sigma_thresh, self.stop_thresh, self.background_brightness)


@NETWORKS.register_module()
class SparseGrid:
    """svox2_network.py:17-162 (constructor) + resample (:320-492), sample (:495-572), save / load (:577-643)."""

    def __init__(self, reso=128, radius=1.0, center=(0.0, 0.0, 0.0), basis_type=BASIS_TYPE_SH, basis_dim=9, basis_reso=16, use_z_order=False,
                 use_sphere_bound=False, mlp_posenc_size=0, mlp_width=16, background_nlayers=0, background_reso=256, device="cuda"):
        if basis_type != BASIS_TYPE_SH:
            raise NotImplementedError(f"SparseGrid: basis_type {basis_type} is not supported; only the SH basis (1) is")
        if basis_dim != 9:
            raise NotImplementedError(f"SparseGrid: basis_dim {basis_dim} is not supported; the kernels run SH of degree 2 (9)")
        if background_nlayers > 0:
            raise NotImplementedError("SparseGrid: the background MSI model (background_nlayers > 0) is not supported")
        self.basis_type, self.basis_dim, self.basis_reso = basis_type, basis_dim, basis_reso
        self.background_nlayers, self.device = 0, device
        reso = [int(reso)] * 3 if np.isscalar(reso) else [int(r) for r in reso]
        assert len(reso) == 3, "reso must be an integer or indexable object of 3 ints"
        if use_z_order and not (reso[0] == reso[1] == reso[2] and reso[0] & (reso[0] - 1) == 0):
            print("Morton code requires a cube grid of power-of-2 size, ignoring...")
            use_z_order = False
        radius = [float(radius)] * 3 if np.isscalar(radius) else [float(r) for r in radius]
        self._radius = torch.tensor(radius, dtype=torch.float32)
        self._center = torch.tensor([float(c) for c in center], dtype=torch.float32)
        self._offset = 0.5 * (1.0 - self._center / self._radius)
        self._scaling = 0.5 / self._radius
        n3 = reduce(lambda x, y: x * y, reso)
        init_links = gen_morton(reso[0]).reshape(-1) if use_z_order else np.arange(n3, dtype=np.int64)
        if use_sphere_bound:
            f = np.float32
            axes = [np.arange(r, dtype=f) - f(0.5) for r in reso]
            gsz = np.array(reso, f)
            pts = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
            pts = (f(1.0) / gsz - f(1.0)) + pts * (f(2.0) / gsz)
            mask = np.linalg.norm(pts, axis=-1) <= f(1.0) + f(3 ** 0.5) / gsz.max()
            self.capacity = int(mask.sum())
            data_mask = np.zeros(n3, np.int64)
            idxs = init_links[mask]
            data_mask[idxs] = 1
            data_mask = np.cumsum(data_mask) - 1
            init_links = np.where(mask, data_mask[init_links], -1)
        else:
            self.capacity = n3
        self._links = torch.from_numpy(init_links.astype(np.int32).reshape(reso)).to(device)
        self.density_data = torch.zeros((self.capacity, 1), dtype=torch.float32, device=device)
        self.sh_data = torch.zeros((self.capacity, 3 * basis_dim), dtype=torch.float32, device=device)
        self.opt = RenderOptions()

    @property
    def use_background(self):
        return False

    def param_init(self, args):
        """svox2_network.py:169-173."""
        self.sh_data.zero_()
        self.density_data.fill_(0.0 if (args.lr_fg_begin_step or 0) > 0 else float(args.init_sigma))

    def setup_render_opts(self, args):
        """svox2_network.py:175-188 (the reference's runner never calls it)."""
        if args.use_spheric_clip:
            raise NotImplementedError("SparseGrid: use_spheric_clip is not supported")
        if args.last_sample_opaque:
            raise NotImplementedError("SparseGrid: last_sample_opaque is not supported")
        if args.random_sigma_std and args.enable_random:
            raise NotImplementedError("SparseGrid: randomized sigma noise is not supported")
        o = self.opt
        o.step_size, o.sigma_thresh, o.stop_thresh = float(args.step_size), float(args.sigma_thresh), float(args.stop_thresh)
        o.background_brightness, o.near_clip = float(args.background_brightness), float(args.near_clip or 0.0)
        if o.near_clip != 0.0:
            raise NotImplementedError("SparseGrid: near_clip != 0 is not supported")

    def xform(self):
        """World -> grid coordinates of the kernels: offset[3] + scaling[3] (volume_render_cuvol.py:33-35, gsz = links.shape[0])."""
        gsz = np.float32(self._links.shape[0])
        return np.concatenate([self._offset.numpy() * gsz - np.float32(0.5), self._scaling.numpy() * gsz]).astype(np.float32)

    # ------------------------------------------------------------------------------------------ rendering
    @torch.no_grad()
    def volume_render_image(self, cam, chunk=1 << 18):
        """(H, W, 3) image of cam (a Camera) in chunks of `chunk` pixels, one launch each and no host synchronisation."""
        n = cam.width * cam.height
        out = torch.empty((n, 3), dtype=torch.float32, device=self._links.device)
        xf, op = self.xform(), self.opt.as_array()
        for s in range(0, n, chunk):
            m = min(chunk, n - s)
            ops.svox_render(m, s, cam.width, cam.c2w, cam.intrin(), self._links, self.density_data, self.sh_data, xf, op, out=out[s:s + m])
        return out.view(cam.height, cam.width, 3)

    # ------------------------------------------------------------------------------------------ resampling
    def sample(self, points, grid_coords=True, want_colors=True):
        """Trilerp at points (N, 3): (density (N, 1), sh (N, 27) or an empty (0, 27)).  Only grid coordinates are supported."""
        if not grid_coords:
            raise NotImplementedError("SparseGrid.sample: only grid coordinates (grid_coords=True) are supported")
        d, s = ops.svox_sample(points.contiguous(), self._links, self.density_data, self.sh_data, want_colors)
        return d.view(-1, 1), (s if want_colors else self.sh_data[:0])

    @torch.no_grad()
    def resample(self, reso, sigma_thresh=5.0, weight_thresh=0.01, dilate=2, cameras=None, use_z_order=False, accelerate=True,
                 weight_render_stop_thresh=0.2, max_elements=0, batch_size=1 << 22):
        """svox2_network.py:320-492: density at the new cells' centres, the keep mask from the max render weight over `cameras`
        (Camera list) or from the density, the top-k bound of max_elements, `dilate` dilations, then links by a scan and SH at the kept
        centres.  Leaves capacity, density_data, sh_data and _links replaced."""
        if use_z_order:
            raise NotImplementedError("SparseGrid.resample: use_z_order is not supported (the reference's runner does not use it)")
        reso = [int(reso)] * 3 if np.isscalar(reso) else [int(r) for r in reso]
        dev = self._links.device
        curr = self._links.shape
        f = np.float32
        lattice = []
        for i in range(3):
            fac = f(0.5 * curr[i] / reso[i])
            start, end = f(fac - f(0.5)), f(f(curr[i]) - fac - f(0.5))
            lattice.append((start, f((end - start) / f(max(reso[i] - 1, 1)))))
        start = np.array([l[0] for l in lattice], f)
        step = np.array([l[1] for l in lattice], f)
        axes = [torch.tensor(start[i], device=dev) + torch.arange(reso[i], dtype=torch.float32, device=dev) * torch.tensor(step[i], device=dev)
                for i in range(3)]
        dense = torch.empty(reso, dtype=torch.float32, device=dev)
        slab = max(1, batch_size // (reso[1] * reso[2]))
        yz = torch.stack(torch.meshgrid(axes[1], axes[2], indexing="ij"), -1).reshape(-1, 2)
        for x0 in range(0, reso[0], slab):
            xs = axes[0][x0:x0 + slab]
            pts = torch.cat([xs.repeat_interleave(yz.shape[0])[:, None], yz.repeat(xs.shape[0], 1)], -1).contiguous()
            dense[x0:x0 + slab] = self.sample(pts, want_colors=False)[0].view(-1, reso[1], reso[2])
        if cameras is not None:
            gsz = f(reso[0])
            xf = np.concatenate([self._offset.numpy() * gsz - f(0.5), self._scaling.numpy() * gsz]).astype(f)
            score = torch.zeros(reso, dtype=torch.float32, device=dev)
            for cam in cameras:
                ops.svox_weight_render(dense, cam.width, cam.height, cam.c2w, cam.intrin(), xf, 0.5, weight_render_stop_thresh, score)
            thresh = weight_thresh
        else:
            score, thresh = dense, sigma_thresh
        mask = score >= thresh
        if max_elements > 0 and max_elements < score.numel() and max_elements < int(mask.sum()):
            bounded = float(torch.topk(score.view(-1), k=max_elements, sorted=False)[0].min())
            thresh = max(thresh, bounded)
            print(" Readjusted threshold to fit to memory:", thresh)
            mask = score >= thresh
        mask = mask.to(torch.uint8).contiguous()
        for _ in range(int(dilate)):
            mask = ops.svox_dilate(mask)
        cap = int(mask.sum())
        links, dens, pts = ops.svox_compact(mask, dense, np.concatenate([start, step]), cap)
        _, sh = self.sample(pts, want_colors=True) if cap else (None, torch.zeros((0, 27), dtype=torch.float32, device=dev))
        self.capacity = cap
        self.density_data = dens.view(-1, 1)
        self.sh_data = sh
        self._links = links

    # ------------------------------------------------------------------------------------------ checkpoint
    def save(self, path, compress=False):
        """svox2_network.py:577-594: np.savez of radius, center, links, density_data (fp32), sh_data (fp16), basis_type."""
        (np.savez_compressed if compress else np.savez)(
            path, radius=self._radius.numpy(), center=self._center.numpy(), links=self._links.cpu().numpy(),
            density_data=self.density_data.cpu().numpy(), sh_data=self.sh_data.cpu().numpy().astype(np.float16), basis_type=self.basis_type)

    @classmethod
    def load(cls, path, device="cuda"):
        """svox2_network.py:596-643 (without the background and learned bases it refuses)."""
        z = np.load(path)
        if "data" in z.files:
            sh_data, density_data = z["data"][..., 1:], z["data"][..., :1]
        else:
            sh_data, density_data = z["sh_data"], z["density_data"]
        if "background_data" in z.files:
            raise NotImplementedError("SparseGrid.load: checkpoints with a background model are not supported")
        radius = z["radius"].tolist() if "radius" in z.files else [1.0, 1.0, 1.0]
        center = z["center"].tolist() if "center" in z.files else [0.0, 0.0, 0.0]
        basis_type = int(z["basis_type"]) if "basis_type" in z.files else BASIS_TYPE_SH
        grid = cls(1, radius=radius, center=center, basis_dim=sh_data.shape[1] // 3, basis_type=basis_type, device=device)
        grid.sh_data = torch.from_numpy(np.ascontiguousarray(sh_data, np.float32)).to(device)
        grid.density_data = torch.from_numpy(np.ascontiguousarray(density_data, np.float32).reshape(-1, 1)).to(device)
        grid._links = torch.from_numpy(np.ascontiguousarray(z["links"], np.int32)).to(device)
        grid.capacity = grid.sh_data.shape[0]
        return grid


class Camera:
    """svox2_utils.py:383-461: OpenCV camera-to-world c2w as 12 device floats, pinhole intrinsics, image size."""

    def __init__(self, c2w, fx, fy, cx, cy, width, height):
        self.c2w, self.fx, self.fy, self.cx, self.cy, self.width, self.height = c2w, fx, fy, cx, cy, int(width), int(height)

    def intrin(self):
        return (self.fx, self.fy, self.cx, self.cy)


class _SvoxImages:
    """The device half of the dataset: uint8 RGBA images (n * H * W, 4), c2w (n, 12) row-major OpenCV camera-to-world (translations
    scaled by scene_scale), one focal length, the principal point at the centre.  Training rays are made in the kernels from pixel ids."""

    def _finish_init(self, split, epoch_size, c2w_opengl, images, focal, scene_scale, device):
        self.split, self.epoch_size, self.scene_scale = split, epoch_size, scene_scale
        self.ndc_coeffs, self.use_sphere_bound = (-1, -1), True
        self.scene_center, self.scene_radius = [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]
        m = np.asarray(c2w_opengl, np.float32) @ np.diag(np.array([1, -1, -1, 1], np.float32))        # OpenGL -> OpenCV
        m[:, :3, 3] *= np.float32(scene_scale)
        self.c2w = torch.from_numpy(np.ascontiguousarray(m)).to(device)
        self.c2w_rows = torch.from_numpy(np.ascontiguousarray(m[:, :3, :4].reshape(-1, 12))).to(device)
        self.n_images, self.h, self.w = images.shape[0], images.shape[1], images.shape[2]
        self.h_full, self.w_full = self.h, self.w
        self.images = images.reshape(-1, 4).contiguous()
        self.focal = float(focal)
        self.intrins = {"fx": self.focal, "fy": self.focal, "cx": self.w * 0.5, "cy": self.h * 0.5}
        self.n_rays = self.n_images * self.h * self.w

    def get_image_size(self, i):
        return self.h, self.w

    def camera(self, i):
        return Camera(self.c2w_rows[i], self.focal, self.focal, self.w * 0.5, self.h * 0.5, self.w, self.h)

    def gt_image(self, i):
        """(H, W, 3) image i composited on white as svox_dataset.py:155-160 does."""
        im = self.images[i * self.h * self.w:(i + 1) * self.h * self.w].float() / 255.0
        return (im[:, :3] * im[:, 3:] + (1.0 - im[:, 3:])).view(self.h, self.w, 3)


@DATASETS.register_module()
class SvoxNeRFDataset(_SvoxImages):
    """svox_dataset.py:94-190: NeRF-synthetic transforms_<split>.json + <split>/<basename>.png, poses OpenGL -> OpenCV, translations times
    scene_scale (2/3), focal 0.5 W / tan(0.5 camera_angle_x), images composited on white (white_bkgd)."""

    def __init__(self, root, split, epoch_size=None, scene_scale=None, factor=1, scale=None, white_bkgd=True, n_images=None, device="cuda", **kwargs):
        from PIL import Image
        assert os.path.isdir(root), f"'{root}' is not a directory"
        if factor != 1 or (scale is not None and scale < 1.0):
            raise NotImplementedError("SvoxNeRFDataset: downscaled images (factor != 1, scale < 1) are not supported")
        scene_scale = 2 / 3 if scene_scale is None else scene_scale
        split_name = split if split != "test_train" else "train"
        with open(os.path.join(root, "transforms_" + split_name + ".json")) as fh:
            j = json.load(fh)
        mats, imgs = [], []
        for frame in j["frames"]:
            im = np.asarray(Image.open(os.path.join(root, split_name, os.path.basename(frame["file_path"]) + ".png")))
            if im.ndim == 2:
                im = im[..., None].repeat(3, -1)
            if im.shape[-1] == 3 or not white_bkgd:
                im = np.concatenate([im[..., :3], np.full(im.shape[:2] + (1,), 255, np.uint8)], -1)
            mats.append(np.array(frame["transform_matrix"], np.float32))
            imgs.append(im)
        if n_images is not None:
            mats, imgs = mats[:n_images], imgs[:n_images]
        focal = float(0.5 * imgs[0].shape[1] / np.tan(0.5 * j["camera_angle_x"]))
        self._finish_init(split, epoch_size, np.stack(mats), torch.from_numpy(np.stack(imgs)).to(device), focal, scene_scale, device)


@DATASETS.register_module()
class SyntheticSvoxDataset(_SvoxImages):
    """SvoxNeRFDataset on the procedural stand-in of the lego scene: SyntheticNerfDataset's cameras (NeRF camera-to-world) and images."""

    def __init__(self, split, epoch_size=None, root=None, n_images=100, H=800, W=800, seed=0, scene_scale=None, device="cuda", **kwargs):
        from .dataset import SyntheticNerfDataset
        ds = SyntheticNerfDataset(batch_size=1, mode="train" if split == "train" else "test", n_images=n_images, H=H, W=W, seed=seed)
        images = ds.image_data.reshape(ds.n_images, ds.H, ds.W, 4)
        self._finish_init(split, epoch_size, np.stack(ds.poses), images, ds._focal[0], 2 / 3 if scene_scale is None else scene_scale, device)
