"""Camera paths of the video renderer, in numpy, as NeRF camera-to-world 3x4 matrices: the reference's spherical path
(dataset/camera_path.py) looking at the origin, and the spiral of LLFF / NeRF's load_llff.py for forward-facing captures."""
import numpy as np


def _trans_t(t):
    return np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, t], [0, 0, 0, 1]], np.float32)


def _rot_phi(phi):
    return np.array([[1, 0, 0, 0], [0, np.cos(phi), -np.sin(phi), 0], [0, np.sin(phi), np.cos(phi), 0], [0, 0, 0, 1]], np.float32)


def _rot_theta(th):
    return np.array([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0], [np.sin(th), 0, np.cos(th), 0], [0, 0, 0, 1]], np.float32)


_SWAP = np.array([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], np.float32)


def pose_spherical(theta, phi, radius):
    """camera_path.py:4-27: azimuth theta and elevation phi in degrees, distance radius -> (3, 4) float32 camera-to-world."""
    c2w = _trans_t(radius)
    c2w = _rot_phi(phi / 180.0 * np.pi) @ c2w
    c2w = _rot_theta(theta / 180.0 * np.pi) @ c2w
    c2w = _SWAP @ c2w
    return c2w[:-1, :]


def path_spherical(nframe=80):
    """camera_path.py:29-31: nframe poses at elevation -30 degrees, radius 4, azimuth from -180 degrees in equal steps."""
    return [pose_spherical(angle, -30.0, 4.0) for angle in np.linspace(-180, 180, nframe + 1)[:-1]]


def _normalize(x):
    return x / np.linalg.norm(x)


def path_spiral(poses, bounds, n_frames=120, n_rots=2, zrate=0.5):
    """render_path_spiral of NeRF's load_llff.py for a forward-facing capture: n_frames (3, 4) float32 camera-to-world matrices on a
    spiral of n_rots turns around the average camera, every one looking at a focus point in front of it.
    poses (n, 3, 4+) NeRF camera-to-world ([right, up, back | position]) and bounds (n, 2) near / far of the capture, both rescaled as
    LLFFDataset keeps them (LLFFDataset.poses / .bounds).  The average camera has the mean position, the summed viewing axis and the
    summed up vector; the focus depth is 1 / ((1 - dt) / close + dt / inf) with close = 0.9 min(bounds), inf = 5 max(bounds), dt = 0.75;
    the radii are the 90th percentile of |camera positions| per axis, and frame k sits at
    c2w_avg @ (radii * (cos th, -sin th, -sin(zrate th))), th = 2 pi n_rots k / n_frames."""
    if bounds is None or np.size(bounds) == 0:
        raise ValueError("path_spiral needs the near / far bounds of the capture (LLFFDataset.bounds); this dataset carries none")
    poses = np.asarray(poses, np.float64)[:, :3, :4]
    bounds = np.asarray(bounds, np.float64)
    up = _normalize(poses[:, :, 1].sum(0))
    z = _normalize(poses[:, :, 2].sum(0))
    x = _normalize(np.cross(up, z))
    c2w = np.stack([x, np.cross(z, x), z, poses[:, :, 3].mean(0)], 1)          # poses_avg
    close, inf, dt = 0.9 * bounds.min(), 5.0 * bounds.max(), 0.75
    focal = 1.0 / ((1.0 - dt) / close + dt / inf)
    rads = np.percentile(np.abs(poses[:, :, 3]), 90, 0)
    focus = c2w @ np.array([0.0, 0.0, -focal, 1.0])
    out = []
    for th in np.linspace(0.0, 2.0 * np.pi * n_rots, n_frames + 1)[:-1]:
        c = c2w @ np.append(np.array([np.cos(th), -np.sin(th), -np.sin(th * zrate)]) * rads, 1.0)
        zz = _normalize(c - focus)
        xx = _normalize(np.cross(up, zz))
        out.append(np.stack([xx, _normalize(np.cross(zz, xx)), zz, c], 1).astype(np.float32))
    return out
