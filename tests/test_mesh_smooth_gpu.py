"""--mcube_smooth on the H100: the signed distance bit for bit against scipy's EDT, the constrained solve against the oracle (same
iteration count, field within 1e-6, every bound exact, no voxel crossing to the other side), the Gaussian within one fp32 ulp of scipy's
gaussian_filter, the method chosen by resolution, bit-reproducible runs, and an end-to-end smoothed extraction from a briefly trained
lego stand-in."""
import os

import numpy as np
import pytest
import torch
from scipy import ndimage

import mesh_smooth_oracle as mso
from test_mesh_cpu import assert_closed_oriented, sphere_field, torus_field, two_spheres
from test_mesh_gpu import trained  # noqa: F401  (module fixture: the lego stand-in after 400 steps)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def npy(t):
    return t.detach().cpu().numpy()


def step(f):
    """an integer step field, as the density lattice float(int(max(sigma, 0))) is"""
    return np.trunc(np.maximum(f, 0)).astype(np.float32)


def blob_field(n, seed=0):
    g = ndimage.gaussian_filter(np.random.default_rng(seed).standard_normal((n, n, n)), 2.0)
    f = step(g * 60)
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = 0, 0, 0, 0, 0, 0
    return f


def slab_field(n):
    """a half-space: D is linear across it, and the energy test ends the solve before max_iters (at 210 for n = 32)"""
    f = np.zeros((n, n, n), np.float32)
    f[:, :, :n // 2] = 3
    return f


@pytest.fixture(scope="module")
def trained_lattice(ops, trained):  # noqa: F811
    m = trained.model
    return npy(ops.density_lattice(64, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights))


FIELDS = {"sphere33": lambda: step(sphere_field(33, 0.3) * 3), "torus64": lambda: step(torus_field(64) * 2),
          "two_spheres96": lambda: step(two_spheres(96) * 2), "blob64": lambda: blob_field(64, seed=7), "slab32": lambda: slab_field(32)}
NAMES = list(FIELDS) + ["trained64"]


def field_of(name, request):
    return request.getfixturevalue("trained_lattice") if name == "trained64" else FIELDS[name]()


@pytest.mark.parametrize("name", NAMES)
def test_signed_distance_matches_scipy_bit_for_bit(ops, name, request):
    f = field_of(name, request)
    D = mso.signed_distance(f)
    out, info = ops.mesh_smooth(cu(f), "constrained", max_iters=0)
    assert np.array_equal(npy(out), D.astype(np.float32))
    assert info == dict(method="constrained", iterations=0, band_variables=int((np.abs(D) < mso.BAND_RADIUS).sum()))


@pytest.mark.parametrize("name", NAMES)
def test_constrained_matches_oracle(ops, name, request):
    f = field_of(name, request)
    ref, it, M = mso.constrained(f)
    out, info = ops.mesh_smooth(cu(f), "constrained")
    out = npy(out)
    assert info == dict(method="constrained", iterations=it, band_variables=M) and M > 0
    assert np.abs(out.astype(np.float64) - ref).max() <= 1e-6
    D = mso.signed_distance(f)
    pos, _ = mso.band(D)
    lower, upper = mso.bounds(D.ravel()[pos])
    x = out.ravel()[pos]
    assert (x >= lower.astype(np.float32)).all() and (x <= upper.astype(np.float32)).all()     # every bound holds exactly
    B = (f > 0).ravel()
    assert (out.ravel()[B] >= 0).all() and (out.ravel()[~B] <= 0).all()                       # no voxel crosses to the other side
    rest = np.ones(f.size, bool)
    rest[pos] = False
    assert np.array_equal(out.ravel()[rest], D.ravel()[rest].astype(np.float32))               # D outside the band


def ulp_distance(a, b):
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-(2 ** 31)) - ia, ia)                                        # monotone integer order of floats
    ib = np.where(ib < 0, np.int64(-(2 ** 31)) - ib, ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("name", ["tiny5", "sphere33", "blob64", "trained64"])
def test_gaussian_within_one_ulp_of_scipy(ops, name, request):
    f = np.random.default_rng(1).random((5, 5, 5)).astype(np.float32) * 3 if name == "tiny5" else field_of(name, request)
    out, info = ops.mesh_smooth(cu(f), "gaussian")
    assert info == dict(method="gaussian", iterations=0, band_variables=0)
    assert ulp_distance(npy(out), mso.gaussian(f)).max() <= 1


def test_auto_picks_the_method_by_resolution(ops):
    for n, method in ((512, "constrained"), (520, "gaussian")):
        f = cu(step(sphere_field(n, 0.3) * 2))
        out, info = ops.mesh_smooth(f, max_iters=10)
        assert info["method"] == method, n
        del out, f
        torch.cuda.empty_cache()


@pytest.mark.parametrize("method", ["constrained", "gaussian"])
def test_two_runs_are_bit_identical(ops, method):
    f = cu(blob_field(96, seed=3))
    a, ia = ops.mesh_smooth(f, method)
    b, ib = ops.mesh_smooth(f, method)
    assert ia == ib and torch.equal(a, b)


def mean_dihedral(verts, tris):
    """mean angle (radians) between the unit normals of faces that share an edge.  Faces of zero area have no normal and are left out:
    the smoothed field clamps voxels to exactly 0, and marching at 0 puts the vertices of their edges on the lattice point itself."""
    p = verts[tris].astype(np.float64)
    nrm = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    area = np.linalg.norm(nrm, axis=1)
    nrm /= np.maximum(area, 1e-300)[:, None]
    e = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    face = np.tile(np.arange(tris.shape[0]), 3)
    key = np.sort(e, 1).astype(np.int64) @ np.array([1 << 32, 1], np.int64)
    o = np.argsort(key, kind="stable")
    k, fo = key[o], face[o]
    pair = np.flatnonzero(k[1:] == k[:-1])
    a, b = fo[pair], fo[pair + 1]
    ok = (area[a] > 0) & (area[b] > 0)
    cos = np.clip((nrm[a[ok]] * nrm[b[ok]]).sum(1), -1, 1)
    return float(np.arccos(cos).mean())


def test_extract_mesh_smooth_end_to_end(ops, trained, tmp_path):  # noqa: F811
    r = trained
    rng0 = r.sampler.rng.copy()
    plain = r.extract_mesh(str(tmp_path / "plain"), resolution=128)
    r.sampler.rng[:] = rng0
    res = r.extract_mesh(str(tmp_path / "smooth"), resolution=128, mcube_smooth=True)
    assert res["smooth"]["method"] == "constrained" and 10 <= res["smooth"]["iterations"] <= 250 and res["smooth"]["band_variables"] > 0
    assert list(res["stage_ms"])[:3] == ["density_lattice", "smooth", "marching_cubes"]
    assert res["n_tris"] > 1000
    assert_closed_oriented(res["triangles"])
    assert mean_dihedral(res["vertices"], res["triangles"]) < mean_dihedral(plain["vertices"], plain["triangles"])
    for f in ("mesh-origin.ply", "mesh-color.ply"):
        assert os.path.getsize(tmp_path / "smooth" / f) > 0
    assert res["colors"].std() > 0
