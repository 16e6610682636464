"""NerfDataset (mirror of dataset/dataset.py:16-270), LLFFDataset (mirror of dataset/llff_dataset.py: forward-facing captures in the
`poses_bounds.npy` layout) and SyntheticNerfDataset, the stand-in used when the NeRF-synthetic `lego` scene is unavailable (the
reference downloads it at run time, dataset_util.py:101-109); write_synthetic_llff writes a forward-facing stand-in to disk.

All expose what the sampler / runner read: n_images, resolution [W,H], aabb_scale, aabb_range, metadata (n,11),
focal_lengths (n,2), transforms_gpu (n, 3x4 stored column-major = 12 floats, dataset.py:164-165), image_data
(n, H*W, 4), batch_size and __next__() -> (img_ids, rays_o, rays_d, rgba).  With `undistort=True` (NerfDataset, SyntheticNerfDataset) also
distortion (n,4) = every image's (k1, k2, p1, p2), in metadata[:, 0:4] too, and, for a non-zero lens, focal_eff (n,2); otherwise distortion
is None and metadata[:, 0:4] stays 0, as in the reference."""
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


LENS_KEYS = ("k1", "k2", "p1", "p2")


def read_lens(json_data):
    """(k1, k2, p1, p2) of an Instant-NGP transforms.json (a missing key counts as 0).  The radial-tangential model below is all the ray
    kernels invert: a fisheye camera or a non-zero k3 / k4 raises NotImplementedError."""
    model = str(json_data.get("camera_model", ""))
    if json_data.get("is_fisheye", False) or "FISHEYE" in model.upper():
        raise NotImplementedError(f"undistort: fisheye cameras (camera_model {model!r}, is_fisheye {json_data.get('is_fisheye', False)}) are not "
                                  "supported; only the radial-tangential model k1, k2, p1, p2 is")
    for k in ("k3", "k4"):
        if float(json_data.get(k, 0.0)) != 0.0:
            raise NotImplementedError(f"undistort: {k} = {json_data[k]} is not supported; only the radial-tangential model k1, k2, p1, p2 is")
    return tuple(float(json_data.get(k, 0.0)) for k in LENS_KEYS)


def lens_distort(x, y, k):
    """OpenCV's radial-tangential model (k3 = 0) in fp64: undistorted normalised camera coordinates (x right, y down) -> distorted ones,
    the ((u - cx)/fx, (v - cy)/fy) of the pixel (u, v).  csrc/lens.cuh is the device form."""
    k1, k2, p1, p2 = k
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    r2 = x * x + y * y
    rad = 1 + r2 * (k1 + r2 * k2)
    return x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y


def _lens_jacobian(x, y, k):
    k1, k2, p1, p2 = k
    r2 = x * x + y * y
    rad, drad = 1 + r2 * (k1 + r2 * k2), 2 * (k1 + 2 * k2 * r2)
    return (rad + x * x * drad + 2 * p1 * y + 6 * p2 * x, x * y * drad + 2 * p1 * x + 2 * p2 * y,
            rad + y * y * drad + 6 * p1 * y + 2 * p2 * x)                # j11, j12 = j21, j22


def lens_undistort(xd, yd, k, iters=50):
    """The inverse of lens_distort in fp64: Newton's method from the distorted point, run to convergence."""
    xd, yd = np.asarray(xd, np.float64), np.asarray(yd, np.float64)
    x, y = xd.copy(), yd.copy()
    for _ in range(iters):
        fx, fy = lens_distort(x, y, k)
        fx, fy = fx - xd, fy - yd
        j11, j12, j22 = _lens_jacobian(x, y, k)
        det = j11 * j22 - j12 * j12
        sx, sy = (j22 * fx - j12 * fy) / det, (j11 * fy - j12 * fx) / det
        x, y = x - sx, y - sy
        if np.max(np.abs(sx) + np.abs(sy), initial=0.0) < 1e-15:
            break
    return x, y


def check_lens(k, W, H, focal, c, n_angles=512, n_radii=2048):
    """ValueError unless the lens k maps the undistorted plane one to one onto the whole image: along every direction from the optical
    axis, the Jacobian determinant of lens_distort stays positive (fp64) until the distorted point is as far out as the image's farthest
    corner.  A lens that folds over inside the image has pixels with two undistorted directions, and the kernels' Newton solve may land
    on either."""
    xs, ys = (np.array([0.0, W]) - c[0]) / focal[0], (np.array([0.0, H]) - c[1]) / focal[1]
    reach = math.hypot(np.abs(xs).max(), np.abs(ys).max())
    th = np.linspace(0, 2 * math.pi, n_angles, endpoint=False)[:, None]
    r = np.linspace(0, 4 * reach, n_radii)[None, :]
    x, y = r * np.cos(th), r * np.sin(th)
    j11, j12, j22 = _lens_jacobian(x, y, k)
    xd, yd = lens_distort(x, y, k)
    out = np.hypot(xd, yd) >= reach
    first_out = np.where(out.any(1), out.argmax(1), n_radii)                       # first sample of every direction beyond the corner
    inside = np.arange(n_radii)[None, :] <= first_out[:, None]
    named = ", ".join(f"{n} = {v:g}" for n, v in zip(LENS_KEYS, k))
    if (first_out == n_radii).any():
        raise ValueError(f"undistort: the lens ({named}) never reaches the image's farthest corner; it cannot be inverted over the image")
    if ((j11 * j22 - j12 * j12 <= 0) & inside).any():
        raise ValueError(f"undistort: the lens ({named}) folds over inside the {W}x{H} image (its Jacobian determinant reaches 0 before the "
                         "farthest corner); the ray kernels cannot invert it reliably")


def frame_extent(k, W, H, focal, c):
    """(x_lo, x_hi, y_lo, y_hi): the signed extent, in fp64, of the undistorted normalised coordinates of the pixel centres and corners of
    a W x H image with focal lengths `focal`, principal point `c` (pixels) and lens k (None or zeros: a pinhole camera, whose extent is
    that of the image's corners).  check_lens makes the map one to one, so the extremes lie on the image's border: its corners and the
    centres of its outer pixels are solved."""
    if k is None or not any(k):
        return (-c[0] / focal[0], (W - c[0]) / focal[0], -c[1] / focal[1], (H - c[1]) / focal[1])
    cu, cv = np.arange(W + 1.0), np.arange(H + 1.0)                                  # corners
    pu, pv = np.arange(W) + 0.5, np.arange(H) + 0.5                                  # centres
    bu = np.concatenate([cu, cu, np.zeros(H + 1), np.full(H + 1, float(W)), pu, pu, np.full(H, 0.5), np.full(H, W - 0.5)])
    bv = np.concatenate([np.zeros(W + 1), np.full(W + 1, float(H)), cv, cv, np.full(W, 0.5), np.full(W, H - 0.5), pv, pv])
    x, y = lens_undistort((bu - c[0]) / focal[0], (bv - c[1]) / focal[1], k)
    return float(x.min()), float(x.max()), float(y.min()), float(y.max())


def lens_extent(k, W, H, focal, c):
    """(max |x_u|, max |y_u|): the undistorted extent, in fp64, of the pixel centres and corners of a W x H image (frame_extent)."""
    x_lo, x_hi, y_lo, y_hi = frame_extent(k, W, H, focal, c)
    return max(-x_lo, x_hi), max(-y_lo, y_hi)


CAMERA_KEYS = ("w", "h", "fl_x", "fl_y", "camera_angle_x", "camera_angle_y", "cx", "cy", "k1", "k2", "k3", "k4", "p1", "p2", "camera_model",
               "is_fisheye")
MAX_PIXELS = 2 ** 31 - 1               # the shuffle holds int32 pixel ids and the kernels uint32 offsets: a split may have at most this many


def read_focal_lengths(cam, W, H):
    """(fx, fy) of a camera dict by the rules of dataset.py:125-142 (fl_<axis>, else camera_angle_<axis> at that axis's resolution; one
    axis stands in for the other), or None when it names neither."""
    def axis(a, res):                                                                               # dataset.py:125-131
        if "fl_" + a in cam:
            return float(cam["fl_" + a])
        if "camera_angle_" + a in cam:
            return fov_to_focal_length(res, cam["camera_angle_" + a] * 180 / math.pi)
        return 0.0
    x_fl, y_fl = axis("x", W), axis("y", H)
    if x_fl != 0:
        return (x_fl, y_fl if y_fl != 0 else x_fl)
    if y_fl != 0:
        return (y_fl, y_fl)
    return None


def frame_camera(top, frame):
    """The camera keys of one entry of `frames` over those of the json's top level: a key in the frame wins over the same key at the top
    level.  A frame that names a focal length or field of view of an axis (fl_<axis> or camera_angle_<axis>) takes both keys of that axis
    from itself, so that its own camera_angle_x is not overruled by a top-level fl_x."""
    cam = {k: top[k] for k in CAMERA_KEYS if k in top}
    for a in ("x", "y"):
        if ("fl_" + a) in frame or ("camera_angle_" + a) in frame:
            cam.pop("fl_" + a, None)
            cam.pop("camera_angle_" + a, None)
    cam.update({k: frame[k] for k in CAMERA_KEYS if k in frame})
    return cam


class _RayBatcher:
    """Pixel shuffling + device ray generation shared by both datasets (dataset.py:57-66,172-188)."""

    def _set_cameras(self, cams):
        """cams: every image's camera (W, H, fx, fy, cx, cy, lens), lens None or (k1, k2, p1, p2) for the rays.  When they are all one
        camera the dataset is set up exactly as from a top-level camera; otherwise the frames keep their own (frame_cameras)."""
        if all(c == cams[0] for c in cams):
            self.W, self.H, fx, fy, self._cx, self._cy, lens = cams[0]
            self._focal = (fx, fy)
            if lens is not None:
                self._lens = lens
        else:
            self._frames = list(cams)
            self.W, self.H = cams[0][0], cams[0][1]

    def _finish_init(self):
        dev = DEVICE
        self.resolution = [self.W, self.H]
        self.n_images = len(self._xforms)
        xf = np.stack(self._xforms).astype(np.float32)                       # (n,3,4)
        self.transforms_gpu = torch.from_numpy(np.ascontiguousarray(xf.transpose(0, 2, 1)).reshape(self.n_images, 12)).to(dev)
        frames = getattr(self, "_frames", None)                              # per-frame cameras that differ, else None
        self.frame_cameras = frames is not None
        self._wh = np.array([c[:2] for c in frames] if frames else [(self.W, self.H)] * self.n_images, np.int64)
        self._offsets = np.concatenate([[0], np.cumsum(self._wh[:, 0] * self._wh[:, 1])])
        self.total_pixels = int(self._offsets[-1])
        if frames and self.total_pixels > MAX_PIXELS:
            raise ValueError(f"per_frame_cameras: the split has {self.total_pixels} pixels; its pixel ids are int32, so at most {MAX_PIXELS}")
        self.resolutions = torch.from_numpy(self._wh.astype(np.int32)).to(dev)
        self.pixel_offsets = torch.from_numpy(self._offsets.astype(np.int32) if self.total_pixels <= MAX_PIXELS else self._offsets).to(dev)
        md = np.zeros((self.n_images, 11), np.float32)
        self.distortion = None
        if frames:
            md[:, 4] = [c[4] / c[0] for c in frames]                         # the principal point of every frame by its own size
            md[:, 5] = [c[5] / c[1] for c in frames]
            md[:, 6], md[:, 7] = [c[2] for c in frames], [c[3] for c in frames]
            self.focal_lengths = torch.from_numpy(md[:, 6:8].copy()).to(dev)
            lenses = [c[6] for c in frames]
            if lenses[0] is not None:
                md[:, 0:4] = lenses
                self.distortion = torch.from_numpy(md[:, 0:4].copy()).to(dev)
            # the occupancy grid's visibility test (grid_mark_untrained_cams): every frame's signed frustum, rounded outwards to f32
            ext = np.array([frame_extent(c[6], c[0], c[1], c[2:4], c[4:6]) for c in frames], np.float64)
            e32 = ext.astype(np.float32)
            lo = np.array([True, False, True, False])
            e32 = np.where(lo & (e32 > ext), np.nextafter(e32, np.float32(-np.inf)), e32)
            e32 = np.where(~lo & (e32 < ext), np.nextafter(e32, np.float32(np.inf)), e32)
            self.frame_extents = torch.from_numpy(np.ascontiguousarray(e32, np.float32)).to(dev)
        else:
            self.focal_lengths = torch.tensor([self._focal] * self.n_images, dtype=torch.float32, device=dev)
            md[:, 4], md[:, 5] = self._cx / self.W, self._cy / self.H
            md[:, 6], md[:, 7] = self._focal
            lens = getattr(self, "_lens", None)                              # (k1, k2, p1, p2) with undistort=True, else None
            if lens is not None:
                md[:, 0:4] = lens                                            # the reference's slots (dataset.py:123-126)
                self.distortion = torch.tensor([lens] * self.n_images, dtype=torch.float32, device=dev)
                if any(lens):
                    # the occupancy grid's visibility frustum (grid_mark_untrained) is symmetric, |x| < (W/2) / f: with these focal lengths
                    # it holds every direction a pixel of the capture sees through the lens
                    ex, ey = lens_extent(lens, self.W, self.H, self._focal, (self._cx, self._cy))
                    self.focal_eff = torch.tensor([[self.W / 2 / ex, self.H / 2 / ey]] * self.n_images, dtype=torch.float32, device=dev)
        self.metadata = torch.from_numpy(md).to(dev)
        self.principal = self.metadata[:, 4:6].contiguous()
        self.aabb_range = (0.5 - self.aabb_scale / 2, 0.5 + self.aabb_scale / 2)    # dataset.py:155-156
        self.idx_now = 0
        self._gen = torch.Generator(device=dev).manual_seed(int(self.seed))
        self.shuffle_index = torch.randperm(self.total_pixels, device=dev, generator=self._gen).int()

    def image_resolution(self, img_id):
        """(W, H) of image img_id."""
        w, h = self._wh[int(img_id)]
        return int(w), int(h)

    def image_pixels(self, img_id):
        """The global pixel ids of image img_id, row-major (int32): its rows of image_data.reshape(-1, 4)."""
        w, h = self.image_resolution(img_id)
        return torch.arange(w * h, device=DEVICE, dtype=torch.int32) + int(self._offsets[int(img_id)])

    def next_pixels(self, n=None):
        """The next n entries of the shuffled pixel list; the list is reshuffled in place when it runs out."""
        n = self.batch_size if n is None else n
        if self.idx_now + n >= self.shuffle_index.shape[0]:
            self.shuffle_index.copy_(torch.randperm(self.total_pixels, device=DEVICE, generator=self._gen).int())
            self.idx_now = 0
        start = self.idx_now
        self.idx_now += n
        return self.shuffle_index[start:start + n]

    def rays_for(self, pix, distortion=None):
        """(img_ids, rays_o, rays_d) of the flat pixel indices pix, through the dataset's lens (or `distortion`) when it has one."""
        distortion = self.distortion if distortion is None else distortion
        lens = {} if distortion is None else dict(distortion=distortion)
        if self.frame_cameras:
            return ops.raygen_cams(pix.contiguous(), self.pixel_offsets, self.resolutions, self.transforms_gpu, self.focal_lengths, self.principal,
                                   **lens)
        return ops.raygen(pix.contiguous(), self.W, self.H, self.transforms_gpu, self.focal_lengths, self.principal, **lens)

    def rgba_for(self, pix):
        v = self.image_data.reshape(-1, 4)[pix.long()]
        return v.float() / 255.0 if v.dtype == torch.uint8 else v

    def __next__(self):
        pix = self.next_pixels()
        img_ids, rays_o, rays_d = self.rays_for(pix)
        return img_ids, rays_o, rays_d, self.rgba_for(pix)

    def generate_rays_total_test(self, img_id):
        """All rays of one image in row-major pixel order (dataset.py:214-238)."""
        _, o, d = self.rays_for(self.image_pixels(img_id))
        return o, d


@DATASETS.register_module()
class NerfDataset(_RayBatcher):
    def __init__(self, root_dir, batch_size, mode="train", H=0, W=0, correct_pose=(1, -1, -1), aabb_scale=None, scale=None, offset=None,
                 img_alpha=True, to_jt=True, have_img=True, preload_shuffle=True, seed=0, undistort=False, per_frame_cameras=False):
        """undistort: read k1, k2, p1, p2 from the split's json and make every ray of its images through that lens (check_lens); off,
        as in the reference, every ray is a pinhole ray.
        per_frame_cameras: every entry of `frames` may carry its own w, h, fl_x, fl_y, camera_angle_x / _y, cx, cy (and, with undistort,
        lens), over the json's top level (frame_camera); images of different sizes are kept in one ragged (total_pixels, 4) table.  When
        the frames resolve to one camera the dataset is the one the top-level keys give.  Off, as in the reference, frame keys are
        ignored."""
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
        cams = []
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
            if per_frame_cameras:
                cams.append(self._frame_camera(json_data, fr, im, W, H, undistort))
            imgs.append(im)
            self.poses.append(np.array(fr["transform_matrix"], np.float32))                           # NeRF camera-to-world, as in the file
            self._xforms.append(matrix_nerf2ngp(fr["transform_matrix"], self.scale, self.offset, correct_pose))
        self.aabb_scale = json_data.get("aabb_scale", 1) if aabb_scale is None else aabb_scale
        self.have_img = have_img
        if per_frame_cameras:
            self._set_cameras(cams)
            if hasattr(self, "_frames"):
                self.image_data = torch.from_numpy(np.concatenate([im.reshape(-1, 4) for im in imgs])).to(DEVICE)
            else:
                self.image_data = torch.from_numpy(np.stack(imgs)).to(DEVICE).reshape(len(imgs), -1, 4)
            self._finish_init()
            return
        self.image_data = torch.from_numpy(np.stack(imgs)).to(DEVICE).reshape(len(imgs), -1, 4)
        self._focal = read_focal_lengths(json_data, self.W, self.H)
        if self._focal is None:
            raise RuntimeError("Couldn't read fov.")
        self._cx, self._cy = json_data.get("cx", self.W / 2), json_data.get("cy", self.H / 2)
        if undistort:
            self._lens = read_lens(json_data)
            check_lens(self._lens, self.W, self.H, self._focal, (self._cx, self._cy))
        self._finish_init()

    @staticmethod
    def _frame_camera(json_data, fr, im, W, H, undistort):
        """(W, H, fx, fy, cx, cy, lens) of one frame (frame_camera); lens is None unless undistort.  The refusals of the lens apply to
        every frame at its own size, and a frame without a resolvable focal length raises."""
        name = fr.get("file_path")
        cam = frame_camera(json_data, fr)
        w = int(cam["w"]) if "w" in cam else (int(W) or im.shape[1])
        h = int(cam["h"]) if "h" in cam else (int(H) or im.shape[0])
        if im.shape[:2] != (h, w):
            raise ValueError(f"per_frame_cameras: frame {name!r} is {im.shape[1]}x{im.shape[0]} pixels but its camera is {w}x{h}")
        f = read_focal_lengths(cam, w, h)
        if f is None:
            raise RuntimeError(f"Couldn't read fov of frame {name!r}: neither it nor the json's top level has fl_x, fl_y, camera_angle_x "
                               "or camera_angle_y")
        c = (cam.get("cx", w / 2), cam.get("cy", h / 2))
        lens = None
        if undistort:
            try:
                lens = read_lens(cam)
                check_lens(lens, w, h, f, c)
            except (NotImplementedError, ValueError) as e:
                raise type(e)(f"frame {name!r}: {e}") from e
        return (w, h, f[0], f[1], c[0], c[1], lens)


def _normalize(x):
    return x / np.linalg.norm(x)


def _viewmatrix(z, up, pos):
    """dataset_util.py:92-98: camera-to-world [x, y, z | pos] looking along z with `up` roughly upwards."""
    z = _normalize(z)
    x = _normalize(np.cross(up, z))
    return np.stack([x, _normalize(np.cross(z, x)), z, pos], 1)


def _poses_avg(poses):
    """llff_dataset.py:181-190: the mean camera (3x5) of (n,3,5) poses -- mean position, summed viewing and up axes."""
    c2w = _viewmatrix(poses[:, :3, 2].sum(0), poses[:, :3, 1].sum(0), poses[:, :3, 3].mean(0))
    return np.concatenate([c2w, poses[0, :3, -1:]], 1)


def _recenter_poses(poses):
    """llff_dataset.py:167-179: all cameras expressed in the frame of the mean camera."""
    out = poses + 0
    bottom = np.reshape([0, 0, 0, 1.0], [1, 4])
    c2w = np.concatenate([_poses_avg(poses)[:3, :4], bottom], -2)
    full = np.concatenate([poses[:, :3, :4], np.tile(bottom[None], [poses.shape[0], 1, 1])], -2)
    out[:, :3, :4] = (np.linalg.inv(c2w) @ full)[:, :3, :4]
    return out


def _image_files(d):
    return [os.path.join(d, f) for f in sorted(os.listdir(d)) if f.endswith(("JPG", "jpg", "png"))]                 # llff_dataset.py:213-214


@DATASETS.register_module()
class LLFFDataset(_RayBatcher):
    """Forward-facing captures as LLFF / COLMAP `imgs2poses` writes them: root_dir/poses_bounds.npy (n,17) and root_dir/images_{factor}
    (or root_dir/images, reduced in memory when the former is missing).  Nothing is written into root_dir (DESIGN.md section 7)."""

    def __init__(self, root_dir, batch_size, mode="train", factor=4, llffhold=0, recenter=True, bd_factor=.75, spherify=False,
                 correct_pose=(1, -1, -1), aabb_scale=None, scale=None, offset=None, img_alpha=True, to_jt=True, have_img=True,
                 preload_shuffle=True, seed=0):
        from PIL import Image
        assert mode in ("train", "val", "test")
        if not isinstance(factor, int) or isinstance(factor, bool) or factor < 1:
            raise ValueError(f"LLFFDataset: factor must be a positive integer, got {factor!r}")                      # llff_dataset.py:48,204-206
        self.root_dir, self.batch_size, self.mode, self.seed = root_dir, batch_size, mode, seed
        self.scale, self.offset = NERF_SCALE, [0.5, 0.5, 0.5]          # the `scale` / `offset` arguments are discarded (llff_dataset.py:24-25)
        self.correct_pose = tuple(correct_pose)
        self.have_img = have_img                                        # images are read whatever this says (llff_dataset.py:91-94)
        # `spherify` is accepted and ignored, as in the reference (its load_data never reads it)
        if aabb_scale is None:
            print("llff dataset need set aabbscale in config file ,automatically set to 32")                          # llff_dataset.py:32-34
            aabb_scale = 32
        self.aabb_scale = aabb_scale
        arr = np.load(os.path.join(root_dir, "poses_bounds.npy"))
        poses = arr[:, :-2].reshape([-1, 3, 5]).transpose([1, 2, 0])                                                  # (3,5,n), :195
        bds = arr[:, -2:].transpose([1, 0])                                                                           # (2,n), :196
        imgdir = os.path.join(root_dir, f"images_{factor}")
        reduce_here = not os.path.isdir(imgdir)                         # the reference runs ImageMagick inside root_dir then (:229-275)
        files = _image_files(os.path.join(root_dir, "images") if reduce_here else imgdir)
        if poses.shape[-1] != len(files):
            raise ValueError(f"LLFFDataset: {len(files)} images in {os.path.dirname(files[0]) if files else root_dir} but "
                             f"{poses.shape[-1]} poses in poses_bounds.npy")

        def read(path):
            im = Image.open(path)
            if reduce_here and factor > 1:
                im = im.resize((int(round(im.width / factor)), int(round(im.height / factor))), Image.BOX)
            im = np.asarray(im)
            if im.ndim == 2:
                im = im[..., None].repeat(3, -1)
            if img_alpha and im.shape[-1] == 3:                                                                       # :130-132
                im = np.concatenate([im, np.full(im.shape[:2] + (1,), 255, np.uint8)], -1)
            return im
        first = read(files[0])
        poses[:2, 4, :] = np.array(first.shape[:2]).reshape([2, 1])                                                   # :221-223
        poses[2, 4, :] = poses[2, 4, :] * 1. / factor
        poses = np.concatenate([poses[:, 1:2, :], -poses[:, 0:1, :], poses[:, 2:, :]], 1)                             # [down,right,back] -> [right,up,back], :139-140
        poses = np.moveaxis(poses, -1, 0).astype(np.float32)
        bds = np.moveaxis(bds, -1, 0).astype(np.float32)
        sc = 1. if bd_factor is None else 1. / (bds.min() * bd_factor)                                                # :147-149
        poses[:, :3, 3] *= sc
        bds *= sc
        if recenter:
            poses = _recenter_poses(poses)
        n = poses.shape[0]
        if llffhold > 0:                                                                                              # :57-59
            i_test = np.arange(n)[::llffhold]
        else:                                                           # the view closest to the mean camera, :155-160
            i_test = np.array([np.argmin(np.sum(np.square(_poses_avg(poses)[:3, 3] - poses[:, :3, 3]), -1))])
        # val is the test set, train is the rest (:60-62); the reference also writes this split to root_dir/split.json
        self.i_select = np.array([i for i in range(n) if i not in i_test]) if mode == "train" else np.asarray(i_test)
        hwf = poses[0, :3, -1]
        self.H, self.W = int(hwf[0]), int(hwf[1])                                                                     # :88-90,121-122
        self._focal = (float(hwf[2]), float(hwf[2]))
        self._cx, self._cy = self.W / 2, self.H / 2                                                                   # :106-107
        poses = poses[:, :3, :4].astype(np.float32)
        self.poses = [poses[i].copy() for i in self.i_select]                                  # NeRF camera-to-world, recentred and rescaled
        self.bounds = bds[self.i_select]                                # (n, 2) near / far of each view, rescaled like the poses (path_spiral)
        self._xforms = [matrix_nerf2ngp(p, self.scale, self.offset, self.correct_pose) for p in self.poses]
        imgs = [first if i == 0 else read(files[i]) for i in self.i_select]
        self.image_data = torch.from_numpy(np.stack(imgs)).to(DEVICE).reshape(len(imgs), self.H * self.W, -1)
        self._finish_init()


def write_synthetic_llff(dst, n_images=20, H=378, W=504, factor=None, seed=0, radius=4.0, extent=0.6, obj_scale=2.2, backdrop_radius=8.0):
    """A forward-facing stand-in on disk, in the layout LLFFDataset reads: dst/poses_bounds.npy and dst/images/*.png of H x W pixels (with
    `factor` also dst/images_{factor}, box-reduced).  Cameras sit on a jittered planar grid of half-width `extent` (NeRF world units) at
    `radius` from the scene and all look at it, as in a hand-held forward-facing capture; the images are ray-traced from
    SyntheticNerfDataset.shade with the opaque backdrop of the "fox" style (every pixel has alpha 1), the two bounds of a view are its
    nearest and farthest analytic hit.  Returns the NeRF camera-to-world matrices [right, up, back | t] it wrote (n,3,4)."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    scene = object.__new__(SyntheticNerfDataset)
    scene.scale, scene.obj_scale, scene.backdrop_radius = NERF_SCALE, obj_scale, backdrop_radius
    focal = 0.81 * W                                                    # the field of view of a phone camera (the fern capture: 3260 / 4032)
    p0 = radius * np.array([math.cos(math.radians(20.0)), 0.0, math.sin(math.radians(20.0))])
    fwd0 = -p0 / np.linalg.norm(p0)
    right0 = _normalize(np.cross(fwd0, [0, 0, 1.0]))
    up0 = np.cross(right0, fwd0)
    side = math.ceil(math.sqrt(n_images))
    os.makedirs(os.path.join(dst, "images"), exist_ok=True)
    if factor:
        os.makedirs(os.path.join(dst, f"images_{factor}"), exist_ok=True)
    v, u = torch.meshgrid(torch.arange(H, device=DEVICE), torch.arange(W, device=DEVICE), indexing="ij")
    d_cam = torch.stack([(u.reshape(-1) + 0.5 - W / 2) / focal, (v.reshape(-1) + 0.5 - H / 2) / focal, torch.ones(H * W, device=DEVICE)], -1)
    rows, mats = [], []
    for k in range(n_images):
        g = (np.array([k % side, k // side]) + rng.uniform(-0.3, 0.3, 2)) / max(side - 1, 1) * 2 - 1
        pos = p0 + extent * (g[0] * right0 + g[1] * up0)
        back = _normalize(pos)                                          # the camera looks along -z at the scene centre
        right = _normalize(np.cross(-back, [0, 0, 1.0]))
        up = np.cross(right, -back)
        c2w = np.stack([right, up, back, pos], 1)
        xf = torch.from_numpy(matrix_nerf2ngp(c2w, NERF_SCALE, [0.5, 0.5, 0.5])).to(DEVICE)
        d = torch.nn.functional.normalize(d_cam @ xf[:, :3].T, dim=-1)
        rgba, t = scene.shade(xf[:, 3].expand(H * W, 3).contiguous(), d.contiguous(), return_t=True)
        t = t / NERF_SCALE                                              # NGP units -> NeRF world units
        img = (rgba[:, :3] * 255.0 + 0.5).clamp(0, 255).to(torch.uint8).reshape(H, W, 3).cpu().numpy()
        im = Image.fromarray(img, "RGB")
        im.save(os.path.join(dst, "images", f"image{k:03d}.png"))
        if factor:
            im.resize((int(round(W / factor)), int(round(H / factor))), Image.BOX).save(os.path.join(dst, f"images_{factor}", f"image{k:03d}.png"))
        m = np.concatenate([np.stack([-up, right, back, pos], 1), np.array([[H], [W], [focal]])], 1)      # inverse of llff_dataset.py:139-140
        rows.append(np.concatenate([m.reshape(-1), [float(t.min()), float(t.max())]]))
        mats.append(c2w)
    np.save(os.path.join(dst, "poses_bounds.npy"), np.stack(rows))
    return np.stack(mats)


def write_synthetic_frames(dst, cameras, n_images=20, seed=0, style="lego", lens_keys=True):
    """A capture whose frames carry their own cameras, on disk in the Instant-NGP layout NerfDataset(per_frame_cameras=True) reads:
    dst/{train,test}/r_{i}.png (RGBA, each at its own size) and dst/transforms_{train,test}.json whose top level holds only aabb_scale
    and whose every frame holds its transform_matrix, w, h, fl_x, fl_y, cx, cy (and k1, k2, p1, p2 for a camera with a lens, unless
    lens_keys is False).  The images are SyntheticNerfDataset(cameras=cameras, ...)'s, so the two datasets describe one scene; the test
    split has n_images // 10 views.  Returns {split: that SyntheticNerfDataset}."""
    from PIL import Image
    out = {}
    for split in ("train", "test"):
        ds = SyntheticNerfDataset(batch_size=1, mode=split, n_images=n_images, seed=seed, style=style, cameras=cameras)
        os.makedirs(os.path.join(dst, split), exist_ok=True)
        table = ds.image_data.reshape(-1, 4).cpu().numpy()
        frames = []
        for i in range(ds.n_images):
            c = tuple(cameras[i % len(cameras)])
            w, h = ds.image_resolution(i)
            lo, hi = int(ds._offsets[i]), int(ds._offsets[i + 1])
            Image.fromarray(table[lo:hi].reshape(h, w, 4), "RGBA").save(os.path.join(dst, split, f"r_{i}.png"))
            fr = dict(file_path=f"./{split}/r_{i}", transform_matrix=np.asarray(ds.poses[i], np.float64).tolist(), w=w, h=h,
                      fl_x=float(c[2]), fl_y=float(c[3]), cx=float(c[4]), cy=float(c[5]))
            if lens_keys and len(c) > 6 and c[6] is not None:
                fr.update(zip(LENS_KEYS, (float(v) for v in c[6])))
            frames.append(fr)
        with open(os.path.join(dst, f"transforms_{split}.json"), "w") as fh:
            json.dump(dict(aabb_scale=ds.aabb_scale, frames=frames), fh)
        out[split] = ds
    return out


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
                 root_dir=None, preload_shuffle=True, style="lego", distortion=None, undistort=False, cameras=None):
        """distortion: (k1, k2, p1, p2) of the lens the images are taken through (None: a pinhole camera); undistort: make the rays
        through that lens, as NerfDataset(undistort=True) does with a capture's json.
        cameras: per-frame cameras (W, H, fx, fy, cx, cy[, lens]), image i taken with cameras[i % len(cameras)] (its lens, if given, in
        place of `distortion`), as NerfDataset(per_frame_cameras=True) reads a capture whose frames carry their own cameras; H, W and
        camera_angle_x are then unused."""
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
        capture = None if distortion is None else tuple(float(v) for v in distortion)
        if cameras is not None:
            cams, capture = [], []
            for i in range(n):
                c = tuple(cameras[i % len(cameras)])
                w, h, fx, fy, cx, cy = int(c[0]), int(c[1]), float(c[2]), float(c[3]), float(c[4]), float(c[5])
                k = tuple(float(v) for v in c[6]) if len(c) > 6 and c[6] is not None else None
                if k is not None:
                    check_lens(k, w, h, (fx, fy), (cx, cy))
                capture.append(k or (0.0, 0.0, 0.0, 0.0))
                cams.append((w, h, fx, fy, cx, cy, (k or (0.0, 0.0, 0.0, 0.0)) if undistort else None))
            self._set_cameras(cams)
            self._finish_init()
            self.image_data = self._render_all(capture if any(any(k) for k in capture) else None)
            return
        if capture is not None:
            check_lens(capture, self.W, self.H, self._focal, (self._cx, self._cy))
        if undistort:
            self._lens = capture or (0.0, 0.0, 0.0, 0.0)
        self._finish_init()
        self.image_data = self._render_all(capture)

    # -- analytic renderer (NGP coordinates: world * 0.33 + 0.5, axes cycled like matrix_nerf2ngp) --------------
    def _to_ngp(self, p):
        p = np.asarray(p, np.float32) * self.scale + 0.5
        return p[[1, 2, 0]]

    def _render_all(self, lens=None):
        """The images, every pixel's ray through `lens` (k1, k2, p1, p2, or one such lens per image) when one is given, whatever rays the
        dataset trains on: (n, H*W, 4), or the ragged (total_pixels, 4) table when the frames' cameras differ."""
        out = torch.empty((self.total_pixels, 4), dtype=torch.uint8, device=DEVICE)
        if lens is not None and any(np.ravel(lens)):
            lens = torch.from_numpy(np.array(np.broadcast_to(np.asarray(lens, np.float32), (self.n_images, 4)), order="C")).to(DEVICE)
        else:
            lens = None
        for i in range(self.n_images):
            pix = self.image_pixels(i)
            if lens is None:
                o, d = self.generate_rays_total_test(i)
            else:
                _, o, d = self.rays_for(pix, lens)
            out[pix.long()] = (self.shade(o, d) * 255.0 + 0.5).clamp(0, 255).to(torch.uint8)
        return out if self.frame_cameras else out.reshape(self.n_images, self.H * self.W, 4)

    def shade(self, o, d, return_t=False, return_normal=False):
        """RGBA in [0,1] of the analytic scene along rays (o,d) given in NGP coordinates; with `return_t` also the distance to the
        hit (inf where the ray leaves the scene), with `return_normal` (last) also the unit outward normal of the surface hit, in NGP
        axes (0 where the ray leaves the scene)."""
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
        rgba = torch.cat([rgb, alpha[:, None]], -1)
        out = (rgba,) + ((t_best,) if return_t else ()) + ((nrm,) if return_normal else ())
        return out if len(out) > 1 else rgba


MULTISCALE_LEVELS = 4                  # full, 1/2, 1/4 and 1/8 resolution, as mip-NeRF's multiscale NeRF-synthetic


def synthetic_multicam(split, n_images=100, H=800, W=800, seed=0, camera_angle_x=0.6911112070083618):
    """The lego stand-in (SyntheticNerfDataset's cameras and images; val and test share the held-out cameras) as a multiscale capture in
    mip-NeRF's layout: every view at full, 1/2, 1/4 and 1/8 resolution (box filter of the full-resolution RGBA, rounded to uint8), view by
    view.  Returns (metadata of the split: {file_path, cam2world (3x4), width, height, pix2cam, lossmult, near, far} lists, [RGBA uint8
    images]).  pix2cam = diag(1, -1, -1) K^-1 (the y and z flips of a NeRF camera), lossmult = the area ratio 4^level."""
    if H % 8 or W % 8:
        raise ValueError(f"synthetic_multicam: H and W must be multiples of 8, got {H} x {W}")
    ds = SyntheticNerfDataset(batch_size=1, mode="train" if split == "train" else "test", n_images=n_images, H=H, W=W, seed=seed,
                              camera_angle_x=camera_angle_x)
    f = float(ds._focal[0])
    meta = {k: [] for k in ("file_path", "cam2world", "width", "height", "pix2cam", "lossmult", "near", "far")}
    images = []
    full = ds.image_data.reshape(ds.n_images, H, W, 4).cpu().numpy()
    for k in range(ds.n_images):
        for lvl in range(MULTISCALE_LEVELS):
            s = 2 ** lvl
            h, w = H // s, W // s
            im = np.floor(full[k].reshape(h, s, w, s, 4).astype(np.float64).mean((1, 3)) + 0.5).astype(np.uint8)
            K = np.array([[f / s, 0, 0.5 * w], [0, f / s, 0.5 * h], [0, 0, 1.0]])
            meta["file_path"].append(f"{split}/r_{k}" + (f"_d{lvl}" if lvl else "") + ".png")
            meta["cam2world"].append(np.asarray(ds.poses[k], np.float64)[:3, :4].tolist())
            meta["width"].append(w)
            meta["height"].append(h)
            meta["pix2cam"].append((np.diag([1.0, -1.0, -1.0]) @ np.linalg.inv(K)).tolist())
            meta["lossmult"].append(float(s * s))
            meta["near"].append(2.0)
            meta["far"].append(6.0)
            images.append(im)
    return meta, images


def write_synthetic_multicam(dst, n_images=100, H=800, W=800, seed=0, camera_angle_x=0.6911112070083618):
    """Writes the multiscale stand-in of synthetic_multicam to dst in mip-NeRF's layout: {split}/r_{k}.png (full resolution) and
    r_{k}_d{1,2,3}.png, and metadata.json, for train / val / test.  transforms_{split}.json lists the full-resolution views, so Blenders
    reads the same directory as the single-scale capture."""
    from PIL import Image
    all_meta = {}
    for split in ("train", "val", "test"):
        meta, images = synthetic_multicam(split, n_images, H, W, seed, camera_angle_x)
        os.makedirs(os.path.join(dst, split), exist_ok=True)
        for p, im in zip(meta["file_path"], images):
            Image.fromarray(im, "RGBA").save(os.path.join(dst, p))
        all_meta[split] = meta
        frames = [dict(file_path="./" + p[:-len(".png")], transform_matrix=c + [[0.0, 0.0, 0.0, 1.0]])
                  for p, c, lm in zip(meta["file_path"], meta["cam2world"], meta["lossmult"]) if lm == 1.0]
        with open(os.path.join(dst, f"transforms_{split}.json"), "w") as fh:
            json.dump(dict(camera_angle_x=camera_angle_x, frames=frames), fh)
    with open(os.path.join(dst, "metadata.json"), "w") as fh:
        json.dump(all_meta, fh)
