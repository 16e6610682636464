"""ctypes bindings for the mesh-extraction oracle (tests/mesh_oracle.c): the marching-cubes table rule, marching cubes, the largest
edge-connected component and vertex normals, plus the density lattice's positions.  TEST INFRASTRUCTURE: imported by tests/ and
tools/gen_mc_table.py only -- never by the product package.

The library is compiled on first use into the system temporary directory (keyed by the source's hash), so nothing is written into
the repository tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mesh_oracle.c")
MAXT = 5                                    # triangles per marching-cubes case (ORC_MC_MAXT)

_u32, _u64, _f32 = C.c_uint32, C.c_uint64, C.c_float
_lib = None


def _ptr(a):
    assert isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"], "need C-contiguous ndarray"
    return a.ctypes.data_as(C.c_void_p)


def lib():
    global _lib
    if _lib is None:
        src = open(SRC, "rb").read()
        so = os.path.join(tempfile.gettempdir(), f"ngp_mesh_oracle_{os.getuid()}_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-o", tmp, SRC, "-lm"])
            os.replace(tmp, so)                                   # atomic: concurrent test processes never load a partial file
        _lib = C.CDLL(so)
    return _lib


def mc_table():
    """The 256-case table from the oracle's rule: (256, 15) cube-edge ids (-1 padded) and (256,) triangle counts."""
    tri = np.empty((256, 3 * MAXT), np.int8)
    ntri = np.empty(256, np.uint8)
    assert lib().orc_mc_table(_ptr(tri), _ptr(ntri)) == MAXT
    return tri, ntri


def marching_cubes(field, iso=0.5):
    """(N,N,N) f32 field -> vertices (V,3) f32 in the PLY frame, triangles (T,3) int32."""
    f = np.ascontiguousarray(field, np.float32)
    n = f.shape[0]
    assert f.shape == (n, n, n)
    counts = np.zeros(2, np.uint64)
    lib().orc_marching_cubes(_u32(n), _ptr(f), _f32(iso), None, None, _u64(0), _u64(0), _ptr(counts))
    verts = np.empty((int(counts[0]), 3), np.float32)
    tris = np.empty((int(counts[1]), 3), np.int32)
    assert lib().orc_marching_cubes(_u32(n), _ptr(f), _f32(iso), _ptr(verts), _ptr(tris), _u64(verts.shape[0]), _u64(tris.shape[0]),
                                    _ptr(counts)) == 0
    return verts, tris


def mesh_largest_component(verts, tris):
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    vo, to = np.empty_like(verts), np.empty_like(tris)
    counts = np.zeros(2, np.uint64)
    lib().orc_mesh_largest_component(_u64(verts.shape[0]), _u64(tris.shape[0]), _ptr(verts), _ptr(tris), _ptr(vo), _ptr(to), _ptr(counts))
    return vo[:int(counts[0])].copy(), to[:int(counts[1])].copy()


def mesh_vertex_normals(verts, tris):
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    nrm = np.empty_like(verts)
    lib().orc_mesh_vertex_normals(_u64(verts.shape[0]), _u64(tris.shape[0]), _ptr(verts), _ptr(tris), _ptr(nrm))
    return nrm


def lattice_positions(n):
    """Model positions of the density lattice, row (i*N + j)*N + k = (i, j, k) / (N-1), each an IEEE fp32 quotient."""
    c = np.arange(n, dtype=np.float32) / np.float32(n - 1)
    i, j, k = np.meshgrid(c, c, c, indexing="ij")
    return np.stack([i.ravel(), j.ravel(), k.ravel()], 1).astype(np.float32)
