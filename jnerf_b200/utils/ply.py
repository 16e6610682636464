"""Binary little-endian PLY writer for triangle meshes, in the layout the reference writes with plyfile (tools/extract_mesh.py:85-90,
:137-143): vertex `x y z` as float [+ `red green blue` as uchar], face `vertex_indices` as a uchar-counted list of int."""
import numpy as np


def write_ply(path, verts, tris, colors=None):
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    vfields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(verts)}",
            "property float x", "property float y", "property float z"]
    if colors is not None:
        colors = np.ascontiguousarray(colors, np.uint8).reshape(-1, 3)
        assert len(colors) == len(verts)
        vfields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    head += [f"element face {len(tris)}", "property list uchar int vertex_indices", "end_header"]
    vrec = np.empty(len(verts), np.dtype(vfields))                   # packed records, no padding
    vrec["x"], vrec["y"], vrec["z"] = verts[:, 0], verts[:, 1], verts[:, 2]
    if colors is not None:
        vrec["red"], vrec["green"], vrec["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
    frec = np.empty(len(tris), np.dtype([("n", "u1"), ("v", "<i4", (3,))]))
    frec["n"] = 3
    frec["v"] = tris
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())
