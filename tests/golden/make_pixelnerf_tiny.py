"""Writes tests/golden/pixelnerf_tiny.npz from the reference's contrib/pixelnerf/tiny_nerf_data.npz: the first three views (the reference
views of main.py:12) and five held-out views, in the same keys, dtypes and layout.

    python tests/golden/make_pixelnerf_tiny.py <path to tiny_nerf_data.npz>
"""
import os
import sys

import numpy as np

HELD_OUT = [20, 40, 60, 80, 101]

if __name__ == "__main__":
    d = np.load(sys.argv[1])
    keep = [0, 1, 2] + HELD_OUT
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pixelnerf_tiny.npz")
    np.savez_compressed(out, images=d["images"][keep], poses=d["poses"][keep], focal=d["focal"])
    print(out, os.path.getsize(out))
