"""Mesh extraction without a GPU: the oracle's marching cubes, component filter and normals on analytic fields (closed, consistently
oriented meshes of the right topology, volume and normals), the committed marching-cubes table against the oracle's rule, the C ABI's
resolution checks, and the host logic of Runner.extract_mesh through tests/mesh_cpu_backend.py (call order, PLY files, frame, colour rays)."""
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch

import mesh_cpu_backend
import mesh_oracle as mo
import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- analytic fields (lattice index space; inside = value > 0.5; the lattice boundary is below 0.5) ----
def grid_coords(n):
    return np.mgrid[0:n, 0:n, 0:n].astype(np.float32)


def sphere_field(n, r_frac=0.3, centre=None):
    g = grid_coords(n)
    c = np.full(3, n / 2, np.float32) if centre is None else np.asarray(centre, np.float32)
    d = np.sqrt(((g - c[:, None, None, None]) ** 2).sum(0))
    return (r_frac * n - d + 0.5).astype(np.float32)


def torus_field(n, R=0.28, r=0.1):
    g = grid_coords(n) / n - 0.5
    q = np.sqrt(g[0] ** 2 + g[1] ** 2) - R
    return ((r - np.sqrt(q ** 2 + g[2] ** 2)) * n + 0.5).astype(np.float32)


def two_spheres(n, r1=0.18, r2=0.12):
    a = sphere_field(n, r1, (0.3 * n, n / 2, n / 2))
    b = sphere_field(n, r2, (0.72 * n, n / 2, n / 2))
    return np.maximum(a, b)


def random_field(n, seed=0):
    f = np.random.default_rng(seed).random((n, n, n), dtype=np.float32)
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = 0, 0, 0, 0, 0, 0
    return f


def directed_edges(tris):
    return Counter(map(tuple, np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]).tolist()))


def assert_closed_oriented(tris):
    de = directed_edges(tris)
    assert max(de.values()) == 1, "a directed edge is used twice: inconsistent orientation"
    assert all((b, a) in de for (a, b) in de), "an edge is used by one triangle only: the mesh has a crack"
    return len(de) // 2


def euler(verts, tris):
    return verts.shape[0] - assert_closed_oriented(tris) + tris.shape[0]


def signed_volume(verts, tris):
    p0, p1, p2 = (verts[tris[:, c]].astype(np.float64) for c in range(3))
    return float((p0 * np.cross(p1, p2)).sum() / 6)


def cases(field, iso=0.5):
    inside = field > iso
    cs = np.zeros(tuple(s - 1 for s in field.shape), np.int32)
    for c in range(8):
        di, dj, dk = c & 1, (c >> 1) & 1, (c >> 2) & 1
        cs |= inside[di:di + cs.shape[0], dj:dj + cs.shape[1], dk:dk + cs.shape[2]].astype(np.int32) << c
    return cs


# ---- marching cubes -------------------------------------------------------------------------------------
def test_committed_table_is_the_oracle_rule():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mc_table
    assert open(gen_mc_table.OUT).read() == gen_mc_table.render()
    tri, ntri = mo.mc_table()
    assert ntri[0] == 0 and ntri[255] == 0 and ntri.max() == 5
    for m in range(256):
        assert (tri[m, :3 * ntri[m]] >= 0).all() and (tri[m, 3 * ntri[m]:] == -1).all()


@pytest.mark.parametrize("name,field,chi", [("sphere", sphere_field(40), 2), ("torus", torus_field(48), 0), ("two_spheres", two_spheres(48), 4)])
def test_analytic_fields_give_closed_oriented_meshes(name, field, chi):
    v, t = mo.marching_cubes(field)
    assert t.shape[0] > 0 and t.min() >= 0 and t.max() < v.shape[0]
    assert len(np.unique(t)) == v.shape[0]                            # every vertex is used
    assert euler(v, t) == chi, name
    assert signed_volume(v, t) > 0                                     # right-hand normals point out in the PLY frame


def test_random_field_exercises_every_case_and_stays_closed():
    f = random_field(40, seed=3)
    assert len(np.unique(cases(f))) == 256
    v, t = mo.marching_cubes(f)
    assert_closed_oriented(t)
    assert signed_volume(v, t) > 0


def test_sphere_volume_and_frame():
    n = 128
    v, t = mo.marching_cubes(sphere_field(n))
    vol = signed_volume(v, t)
    assert abs(vol / (4 / 3 * np.pi * 0.3 ** 3) - 1) < 0.01
    assert np.abs(v.mean(0) - 0.5).max() < 1e-3                        # lattice position / N: the centre n/2 lands on 0.5


def test_vertex_numbering_and_interpolation():
    """Vertex = lattice edge in (point, axis) order, placed at a + (iso - f_a) / (f_b - f_a) from the lower endpoint, PLY frame."""
    n = 5
    f = np.zeros((n, n, n), np.float32)
    f[2, 2, 2] = 2.0
    v, t = mo.marching_cubes(f)
    # crossing edges, in order: (1,2,2)+x, (2,1,2)+y, (2,2,1)+z, (2,2,2)+x, (2,2,2)+y, (2,2,2)+z
    t_lo = np.float32(0.5) / np.float32(2.0)                          # from the outside endpoint (f = 0) towards f = 2
    t_hi = (np.float32(0.5) - np.float32(2.0)) / (np.float32(0.0) - np.float32(2.0))
    lat = np.array([[1 + t_lo, 2, 2], [2, 1 + t_lo, 2], [2, 2, 1 + t_lo], [2 + t_hi, 2, 2], [2, 2 + t_hi, 2], [2, 2, 2 + t_hi]], np.float32)
    ply = (lat / np.float32(n))[:, [1, 0, 2]]
    assert np.array_equal(v, ply)
    assert t.shape[0] == 8 and euler(v, t) == 2


# ---- component filter / normals ------------------------------------------------------------------------------
def test_largest_component_keeps_the_larger_sphere():
    v, t = mo.marching_cubes(two_spheres(48))
    vk, tk = mo.mesh_largest_component(v, t)
    big, _ = mo.marching_cubes(sphere_field(48, 0.18, (0.3 * 48, 24, 24)))
    assert vk.shape[0] == big.shape[0] and euler(vk, tk) == 2
    assert vk[:, 1].max() < 0.5                                        # PLY y = model x: the sphere at x = 0.3
    assert np.array_equal(np.unique(tk), np.arange(vk.shape[0]))       # compacted, every vertex referenced
    # order kept: the kept vertices are a subsequence of the input, and so are the kept triangles after the index remap
    vpos = {tuple(x): i for i, x in enumerate(v.tolist())}
    idx = np.array([vpos[tuple(x)] for x in vk.tolist()])
    assert (np.diff(idx) > 0).all()
    tpos = {tuple(x): i for i, x in enumerate(t.tolist())}
    assert (np.diff([tpos[tuple(x)] for x in idx[tk].tolist()]) > 0).all()


def test_largest_component_tie_keeps_the_lowest_triangle():
    n = 48
    a = sphere_field(n, 0.12, (14, 24, 24))
    b = sphere_field(n, 0.12, (34, 24, 24))                            # the same sphere 20 cells further along x: same count
    v, t = mo.marching_cubes(np.maximum(a, b))
    vk, tk = mo.mesh_largest_component(v, t)
    assert 2 * tk.shape[0] == t.shape[0]
    assert vk[:, 1].max() < 24 / n                                     # the sphere of the lower cells (PLY y = model x)
    # edge-connected, not vertex-connected: a bow tie of two triangles sharing one vertex is two clusters; the first wins a tie
    bv = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [-1, 0, 0], [0, -1, 0]], np.float32)
    bt = np.array([[0, 3, 4], [0, 1, 2]], np.int32)
    vk, tk = mo.mesh_largest_component(bv, bt)
    assert np.array_equal(tk, [[0, 1, 2]]) and np.array_equal(vk, bv[[0, 3, 4]])


def test_sphere_normals_point_outward():
    n = 64
    v, t = mo.marching_cubes(sphere_field(n))
    nrm = mo.mesh_vertex_normals(v, t)
    radial = v - 0.5
    radial /= np.linalg.norm(radial, axis=1, keepdims=True)
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1, atol=1e-6)
    assert (np.einsum("ij,ij->i", nrm, radial) > 0.99).all()


def test_c_abi_rejects_bad_resolutions():
    from jnerf_b200 import build, lib as L
    build.build()
    lib = L.load()
    counts = np.zeros(2, np.uint64)
    for n in (0, 1, 1025):
        assert lib.ngp_density_lattice(None, n, None, None, None, None) != 0
        assert b"[2, 1024]" in lib.ngp_last_error()
        assert lib.ngp_marching_cubes(None, n, None, 0.5, None, None, 0, None, 0, counts.ctypes.data) != 0
        assert b"[2, 1024]" in lib.ngp_last_error()
    assert lib.ngp_mesh_largest_component(None, 1 << 31, 1, None, None, None, None, None, counts.ctypes.data) != 0
    b = np.zeros(1, np.uint64)
    assert lib.ngp_mesh_workspace_bytes(512, 0, 0, b.ctypes.data) == 0 and int(b[0]) >= 2 * 512 ** 3
    assert lib.ngp_mesh_workspace_bytes(1025, 0, 0, b.ctypes.data) != 0 and b"[2, 1024]" in lib.ngp_last_error()


# ---- Runner.extract_mesh host logic ---------------------------------------------------------------------------
def read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[:2] == ["ply", "format binary_little_endian 1.0"] and head[-1] == "end_header"
    elems, cur = [], None
    for line in head[2:-1]:
        w = line.split()
        if w[0] == "element":
            cur = [w[1], int(w[2]), []]
            elems.append(cur)
        else:
            assert w[0] == "property"
            cur[2].append(tuple(w[1:]))
    (vn, nv, vprops), (fn, nf, fprops) = elems
    assert vn == "vertex" and fn == "face" and fprops == [("list", "uchar", "int", "vertex_indices")]
    types = {"float": "<f4", "uchar": "u1"}
    vdt = np.dtype([(p[1], types[p[0]]) for p in vprops])
    verts = np.frombuffer(data, vdt, nv, end)
    faces = np.frombuffer(data, np.dtype([("n", "u1"), ("v", "<i4", (3,))]), nf, end + nv * vdt.itemsize)
    assert end + nv * vdt.itemsize + nf * 13 == len(data) and (faces["n"] == 3).all()
    return vprops, verts, faces["v"]


def ellipsoid_field(n):
    """A solid elongated along model x (the first lattice index), density 4 inside."""
    g = grid_coords(n) / np.float32(n - 1) - 0.5
    d = (g[0] / 0.38) ** 2 + (g[1] / 0.18) ** 2 + (g[2] / 0.18) ** 2
    return np.where(d < 1, 4.0, 0.0).astype(np.float32)


def test_runner_extract_mesh_on_cpu(monkeypatch, tmp_path):
    from test_runner_cpu import make_runner
    r, fake = make_runner(monkeypatch, rays=64)
    mesh_cpu_backend.install(monkeypatch, fake)
    from jnerf_b200 import ops
    n = 16
    field = ellipsoid_field(n)
    real_lattice = ops.density_lattice
    lat = real_lattice(n, r.model.pos_encoder.m_grid, r.model.pos_encoder.levels, r.model.density_mlp.con_weights)   # the oracle lattice runs
    assert lat.shape == (n, n, n) and (lat >= 0).all() and torch.equal(lat, torch.trunc(lat))
    monkeypatch.setattr(ops, "density_lattice", lambda *a, **k: (fake._log("density_lattice"), torch.from_numpy(field))[1])
    marched = []
    march = ops.march

    def spy(rays_o, rays_d, *a, **k):
        marched.append((rays_o.clone().numpy(), rays_d.clone().numpy()))
        return march(rays_o, rays_d, *a, **k)
    monkeypatch.setattr(ops, "march", spy)
    rng0 = r.sampler.rng.copy()
    fake.calls.clear()
    res = r.extract_mesh(str(tmp_path), resolution=n)
    nb = -(-res["n_verts"] // 64)
    assert fake.calls == ["density_lattice", "marching_cubes", "mesh_largest_component", "mesh_vertex_normals"] + \
        ["march", "network_fwd", "composite_infer"] * nb
    rng = rng0.copy()
    for _ in range(nb):
        rng = ol.pcg32_advance(rng)
    assert np.array_equal(r.sampler.rng, rng)                          # one advance per batch
    # both files parse, with the reference's header, types and counts
    vp, v0, f0 = read_ply(tmp_path / "mesh-origin.ply")
    assert vp == [("float", "x"), ("float", "y"), ("float", "z")]
    assert len(v0) == res["n_verts_origin"] and len(f0) == res["n_tris_origin"]
    vp, v1, f1 = read_ply(tmp_path / "mesh-color.ply")
    assert vp == [("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"), ("uchar", "green"), ("uchar", "blue")]
    assert len(v1) == res["n_verts"] > 0 and len(f1) == res["n_tris"] > 0
    assert np.array_equal(np.stack([v1["x"], v1["y"], v1["z"]], 1), res["vertices"]) and np.array_equal(f1, res["triangles"])
    assert np.array_equal(np.stack([v1["red"], v1["green"], v1["blue"]], 1), res["colors"])
    assert_closed_oriented(res["triangles"])
    # the frame: elongated along model x -> along PLY y
    ext = res["vertices"].max(0) - res["vertices"].min(0)
    assert ext[1] > 1.8 * ext[0] and ext[1] > 1.8 * ext[2]
    # colour rays: from 0.2 outside the vertex (model frame) along the unit normal into the object
    o = np.concatenate([m[0] for m in marched])
    d = np.concatenate([m[1] for m in marched])
    vm = res["vertices"][:, [1, 0, 2]]
    assert np.allclose(o + 0.2 * d, vm, atol=1e-6) and np.allclose(np.linalg.norm(d, axis=1), 1, atol=1e-5)
    c = (n - 1) / (2 * n)                                              # the ellipsoid's centre, index (n-1)/2, in the /N vertex frame
    assert (np.einsum("ij,ij->i", c - vm, d) > 0).all()                # towards the inside
    scale = np.array([0.38, 0.18, 0.18]) * (n - 1) / n
    inside = lambda p: (((p - c) / scale) ** 2).sum(1)                 # noqa: E731
    assert (inside(o) > inside(vm)).all()                              # the origin is on the low-density side


def test_runner_extract_mesh_rejects_bad_resolution(monkeypatch, tmp_path):
    from test_runner_cpu import make_runner
    r, fake = make_runner(monkeypatch, rays=64)
    mesh_cpu_backend.install(monkeypatch, fake)
    for n in (1, 1025):
        with pytest.raises(ValueError, match="2, 1024"):
            r.extract_mesh(str(tmp_path), resolution=n)
