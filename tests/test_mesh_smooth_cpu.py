"""--mcube_smooth without a GPU: the smoothing oracle (tests/mesh_smooth_oracle.py) on cases checked by hand (the operator's diagonal and
rows, the signed distance against a brute-force EDT, the Gaussian against an explicit 25-tap correlation), the C ABI's argument checks,
and the host logic of Runner.extract_mesh(mcube_smooth=True) with the smoothing op computed by the oracle."""
import numpy as np
import pytest
import torch

import mesh_cpu_backend
import mesh_smooth_oracle as mso
from test_mesh_cpu import assert_closed_oriented, ellipsoid_field, read_ply, sphere_field


# ---- the operator -----------------------------------------------------------------------------------------------------------------
def test_operator_on_a_line():
    """Five variables in a chain along k: q_k is the second difference (one-sided at the ends), q_i = q_j = 0."""
    nb = np.full((5, 6), -1, np.int64)
    nb[1:, 4] = np.arange(4)
    nb[:4, 5] = np.arange(1, 5)
    Q = mso.q_matrix(nb).toarray()
    assert np.array_equal(Q[0::3], 0 * Q[0::3]) and np.array_equal(Q[1::3], 0 * Q[1::3])
    assert np.array_equal(Q[2::3], [[-1, 1, 0, 0, 0], [1, -2, 1, 0, 0], [0, 1, -2, 1, 0], [0, 0, 1, -2, 1], [0, 0, 0, 1, -1]])
    A = Q.T @ Q
    assert np.array_equal(A, [[2, -3, 1, 0, 0], [-3, 6, -4, 1, 0], [1, -4, 6, -4, 1], [0, 1, -4, 6, -3], [0, 0, 1, -3, 2]])
    assert np.array_equal(mso.diag_a(nb), np.diag(A))
    x = np.array([0.5, -1.0, 2.0, 0.25, 3.0])
    assert mso.energy(mso.q_matrix(nb), x) == pytest.approx(0.5 * x @ A @ x)


def test_operator_at_a_band_corner():
    """n = 3 with one inside voxel: all 27 voxels are variables.  At the corner (0,0,0) each axis has one neighbour inside the lattice
    (m_a = 1): diag 3 * (1 + 1) = 6, -3 towards the neighbour at 1 (-1 * 1 from q_a(corner), 1 * -2 from q_a(neighbour)), 1 towards 2."""
    f = np.zeros((3, 3, 3), np.float32)
    f[1, 1, 1] = 5
    D = mso.signed_distance(f)
    pos, nb = mso.band(D)
    assert np.array_equal(pos, np.arange(27))
    assert np.array_equal(nb[0], [-1, 9, -1, 3, -1, 1])
    A = (mso.q_matrix(nb).T @ mso.q_matrix(nb)).toarray()
    row = np.zeros(27)
    row[0] = 6
    row[[9, 3, 1]] = -3
    row[[18, 6, 2]] = 1
    assert np.array_equal(A[0], row)
    assert np.array_equal(mso.diag_a(nb), np.diag(A))
    assert mso.diag_a(nb)[13] == 18                                    # the centre: m_a = 0 on every axis, 3 * 6
    # bounds: the centre (x0 = 0.5) gets lower 0, a face neighbour (-0.5) and an edge neighbour (-(sqrt 2 - 0.5)) upper 0,
    # a corner keeps its own -(sqrt 3 - 0.5)
    lower, upper = mso.bounds(D.ravel())
    assert lower[13] == 0 and upper[13] == np.inf
    assert upper[4] == 0 and upper[1] == 0 and upper[0] == -(np.sqrt(3) - 0.5) and lower[0] == -np.inf


def brute_force_sdist(f):
    B = f > 0
    pts = np.argwhere(np.ones(f.shape, bool))
    ins, outs = np.argwhere(B), np.argwhere(~B)
    d_out = ((pts[:, None, :] - outs[None]) ** 2).sum(-1).min(1)       # squared distance to the nearest outside voxel
    d_in = ((pts[:, None, :] - ins[None]) ** 2).sum(-1).min(1)
    return np.where(B.ravel(), np.sqrt(d_out) - 0.5, -np.sqrt(d_in) + 0.5).reshape(f.shape)


@pytest.mark.parametrize("name", ["sphere", "box", "random"])
def test_signed_distance_is_the_exact_edt(name):
    n = 12
    f = {"sphere": lambda: sphere_field(n, 0.3), "box": lambda: np.pad(np.full((5, 7, 3), 2, np.float32), ((2, 5), (1, 4), (4, 5))),
         "random": lambda: (np.random.default_rng(4).random((n, n, n)) > 0.7).astype(np.float32)}[name]()
    D = mso.signed_distance(f)
    assert np.array_equal(D, brute_force_sdist(f))
    k = (np.abs(D) + 0.5) ** 2                                         # every value is +-(sqrt(k) - 0.5), k a positive integer
    assert np.allclose(k, np.round(k), atol=1e-9) and (np.round(k) >= 1).all()
    assert np.array_equal(D > 0, f > 0)


def test_empty_classes_give_a_constant_field():
    for f, v in ((np.zeros((6, 6, 6), np.float32), -1), (np.ones((6, 6, 6), np.float32), 1)):
        out, info = mso.smooth(f)
        assert (out == v).all() and info == dict(method="constrained", iterations=0, band_variables=0)


def test_gaussian_is_the_25_tap_correlation_with_reflect():
    f = np.random.default_rng(2).random((14, 15, 16)).astype(np.float32) * 4
    j = np.arange(-12, 13)
    w = np.exp(-0.5 / 9 * j ** 2)
    w /= w.sum()
    g = f.astype(np.float64) - 0.5
    for a in range(3):
        n = g.shape[a]
        idx = np.arange(n)[:, None] + j[None]
        idx = np.where(idx < 0, -idx - 1, np.where(idx >= n, 2 * n - 1 - idx, idx))   # -1 -> 0, n -> n - 1
        g = np.moveaxis((np.moveaxis(g, a, -1)[..., idx] * w).sum(-1), -1, a)
    assert np.allclose(mso.gaussian(f), g.astype(np.float32), rtol=1e-6, atol=1e-6)


def test_method_selection():
    assert mso.pick_method(512) == "constrained" and mso.pick_method(513) == "gaussian"
    assert mso.pick_method(1024, "constrained") == "constrained" and mso.pick_method(8, "gaussian") == "gaussian"


def test_constrained_keeps_bounds_and_lowers_the_energy():
    f = np.trunc(np.maximum(sphere_field(24, 0.3), 0))                # an integer step field, as the density lattice is
    D = mso.signed_distance(f)
    pos, nb = mso.band(D)
    out, it, M = mso.constrained(f)
    assert M == pos.size and 10 <= it <= mso.MAX_ITERS
    x0, x = D.ravel()[pos], out.ravel()[pos].astype(np.float64)
    lower, upper = mso.bounds(x0)
    xf = mso.constrained(f)[0].ravel()[pos]
    assert np.array_equal(out.ravel()[pos], xf)                         # deterministic
    assert (x >= np.float32(lower)).all() and (x <= np.float32(upper)).all()
    assert np.array_equal(out.ravel()[np.setdiff1d(np.arange(f.size), pos)], D.ravel()[np.setdiff1d(np.arange(f.size), pos)].astype(np.float32))
    Q = mso.q_matrix(nb)
    assert mso.energy(Q, x) < 0.5 * mso.energy(Q, x0)
    assert np.array_equal(mso.constrained(f, 0)[0], D.astype(np.float32))


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
def test_c_abi_rejects_bad_arguments():
    from jnerf_b200 import build, lib as L
    build.build()
    lib = L.load()
    info = np.zeros(3, np.uint32)
    b = np.zeros(1, np.uint64)
    P, Q = 1 << 20, 2 << 20                                            # never dereferenced: every call below is refused first
    for n in (0, 1, 1025):
        assert lib.ngp_mesh_smooth(None, n, P, 0, 250, P, 1 << 40, Q, info.ctypes.data) != 0 and b"[2, 1024]" in lib.ngp_last_error()
        assert lib.ngp_mesh_smooth_workspace_bytes(n, 0, b.ctypes.data) != 0 and b"[2, 1024]" in lib.ngp_last_error()
    assert lib.ngp_mesh_smooth(None, 8, P, 3, 250, P, 1 << 40, Q, info.ctypes.data) != 0 and b"method" in lib.ngp_last_error()
    for args in ((None, P, Q, info.ctypes.data), (P, None, Q, info.ctypes.data), (P, P, None, info.ctypes.data), (P, P, Q, None)):
        field, ws, out, inf = args
        assert lib.ngp_mesh_smooth(None, 8, field, 0, 250, ws, 1 << 40, out, inf) != 0 and b"required" in lib.ngp_last_error()
    assert lib.ngp_mesh_smooth(None, 8, P, 0, 250, P, 1 << 40, P, info.ctypes.data) != 0 and b"separate" in lib.ngp_last_error()
    for method in (0, 1, 2):
        assert lib.ngp_mesh_smooth_workspace_bytes(8, method, b.ctypes.data) == 0
        assert lib.ngp_mesh_smooth(None, 8, P, method, 250, Q + (1 << 20), int(b[0]) - 1, Q, info.ctypes.data) != 0
        assert b"workspace" in lib.ngp_last_error()
    sizes = {}
    for n, method in ((512, 0), (512, 1), (520, 0), (520, 2), (1024, 1)):
        assert lib.ngp_mesh_smooth_workspace_bytes(n, method, b.ctypes.data) == 0
        sizes[n, method] = int(b[0])
    assert sizes[512, 0] == sizes[512, 1] >= 72 * 512 ** 3 and sizes[520, 0] == sizes[520, 2] >= 8 * 520 ** 3
    assert sizes[520, 2] < 9 * 520 ** 3 and sizes[1024, 1] >= 72 * 1024 ** 3


# ---- Runner.extract_mesh host logic -------------------------------------------------------------------------------------------------
def install_smooth(monkeypatch, fake):
    """ops.mesh_smooth computed by the oracle, logged in the fake backend's call list."""
    import jnerf_b200.ops as real_ops
    seen = []

    def mesh_smooth(field, method="auto", max_iters=250, workspace=None):
        fake._log("mesh_smooth")
        f = field.detach().cpu().numpy()
        seen.append(f.copy())
        out, info = mso.smooth(f, method, max_iters)
        return torch.from_numpy(out), info
    monkeypatch.setattr(real_ops, "mesh_smooth", mesh_smooth)
    return seen


def run_extract(monkeypatch, tmp_path, mcube_smooth):
    from test_runner_cpu import make_runner
    from jnerf_b200 import ops
    r, fake = make_runner(monkeypatch, rays=64)
    mesh_cpu_backend.install(monkeypatch, fake)
    seen = install_smooth(monkeypatch, fake)
    n = 16
    field = ellipsoid_field(n)
    monkeypatch.setattr(ops, "density_lattice", lambda *a, **k: (fake._log("density_lattice"), torch.from_numpy(field))[1])
    isos, marched = [], []
    mc = ops.marching_cubes

    def mc_spy(f, iso=0.5, workspace=None):
        isos.append(iso)
        marched.append(f.detach().cpu().numpy().copy())
        return mc(f, iso, workspace)
    monkeypatch.setattr(ops, "marching_cubes", mc_spy)
    fake.calls.clear()
    res = r.extract_mesh(str(tmp_path), resolution=n, mcube_smooth=mcube_smooth)
    return res, fake, field, seen, isos, marched


def test_runner_extract_mesh_smooth_on_cpu(monkeypatch, tmp_path):
    res, fake, field, seen, isos, marched = run_extract(monkeypatch, tmp_path, True)
    nb = -(-res["n_verts"] // 64)
    assert fake.calls == ["density_lattice", "mesh_smooth", "marching_cubes", "mesh_largest_component", "mesh_vertex_normals"] + \
        ["march", "network_fwd", "composite_infer"] * nb
    assert len(seen) == 1 and np.array_equal(seen[0], field)          # the lattice goes to the smoothing ...
    smoothed, info = mso.smooth(field)
    assert isos == [0.0] and np.array_equal(marched[0], smoothed)      # ... and its result is marched at 0
    assert res["smooth"] == info and info["method"] == "constrained" and info["band_variables"] > 0
    assert list(res["stage_ms"]) == ["density_lattice", "smooth", "marching_cubes", "write_origin", "component_normals", "colour"]
    _, v0, f0 = read_ply(tmp_path / "mesh-origin.ply")
    assert len(v0) == res["n_verts_origin"] and len(f0) == res["n_tris_origin"] > 0
    _, v1, f1 = read_ply(tmp_path / "mesh-color.ply")
    assert len(v1) == res["n_verts"] > 0 and np.array_equal(f1, res["triangles"])
    assert_closed_oriented(res["triangles"])


def test_runner_extract_mesh_without_smooth_is_unchanged(monkeypatch, tmp_path):
    res, fake, field, seen, isos, marched = run_extract(monkeypatch, tmp_path, False)
    nb = -(-res["n_verts"] // 64)
    assert fake.calls == ["density_lattice", "marching_cubes", "mesh_largest_component", "mesh_vertex_normals"] + \
        ["march", "network_fwd", "composite_infer"] * nb
    assert not seen and isos == [0.5] and np.array_equal(marched[0], field) and "smooth" not in res
    assert list(res["stage_ms"]) == ["density_lattice", "marching_cubes", "write_origin", "component_normals", "colour"]
