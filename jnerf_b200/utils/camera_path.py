"""The spherical camera path of the video renderer (dataset/camera_path.py of the reference), in numpy: NeRF camera-to-world 3x4
matrices looking at the origin."""
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
