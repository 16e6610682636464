"""The mesh-extraction operators of jnerf_b200/ops.py computed by the mesh oracle (tests/mesh_oracle.py) on CPU tensors, installed on
top of tests/cpu_backend.py so that Runner.extract_mesh's host logic runs without a GPU.  Test infrastructure, like cpu_backend."""
import numpy as np
import torch

import cpu_backend
import mesh_oracle as mo


def _np(t, dtype):
    return np.ascontiguousarray(t.detach().cpu().numpy().astype(dtype, copy=False))


def install(monkeypatch, fake=None):
    """cpu_backend.install (unless `fake` is the OracleOps it returned) + the four mesh operators, logged in the same call list."""
    if fake is None:
        fake = cpu_backend.install(monkeypatch)
    import jnerf_b200.ops as real_ops

    def density_lattice(n, grid, levels, wd):
        fake._log("density_lattice")
        if not 2 <= int(n) <= 1024:
            raise RuntimeError(f"density_lattice: resolution {n} is outside [2, 1024]")
        sig = fake.density_fwd(torch.from_numpy(mo.lattice_positions(n)), grid, levels, wd)   # the oracle's density path
        fake.calls.pop()                                                                       # counted as one operator
        return torch.from_numpy(np.trunc(np.maximum(_np(sig, np.float32), 0)).astype(np.float32).reshape(n, n, n))

    def marching_cubes(field, iso=0.5, workspace=None):
        fake._log("marching_cubes")
        v, t = mo.marching_cubes(_np(field, np.float32), iso)
        return torch.from_numpy(v), torch.from_numpy(t)

    def mesh_largest_component(verts, tris, workspace=None):
        fake._log("mesh_largest_component")
        v, t = mo.mesh_largest_component(_np(verts, np.float32), _np(tris, np.int32))
        return torch.from_numpy(v), torch.from_numpy(t)

    def mesh_vertex_normals(verts, tris, workspace=None):
        fake._log("mesh_vertex_normals")
        return torch.from_numpy(mo.mesh_vertex_normals(_np(verts, np.float32), _np(tris, np.int32)))

    for f in (density_lattice, marching_cubes, mesh_largest_component, mesh_vertex_normals):
        monkeypatch.setattr(real_ops, f.__name__, f)
    return fake
