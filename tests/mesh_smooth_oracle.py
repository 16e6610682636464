"""numpy / scipy restatement of PyMCubes' smooth(sigma) as DESIGN.md section 7 states it: the constrained method (signed distance from
scipy's exact EDT, then the bounded Jacobi solve on the band |D| < 4) and the Gaussian one (scipy's gaussian_filter of f - 0.5, sigma 3).
TEST INFRASTRUCTURE, like tests/mesh_oracle.py: imported by tests/ only, vectorised (no per-voxel Python loop)."""
import numpy as np
from scipy import ndimage, sparse

BAND_RADIUS = 4.0
MAX_ITERS = 250
CHECK_EVERY = 10
REL_TOL = 1e-6
STOP_RATIO = 1 - (1 - REL_TOL) ** CHECK_EVERY
AUTO_MAX_N = 512
METHODS = ("auto", "constrained", "gaussian")


def pick_method(n, method="auto"):
    if method != "auto":
        return method
    return "constrained" if n ** 3 <= AUTO_MAX_N ** 3 else "gaussian"


def signed_distance(f):
    """D = EDT(B) - 0.5 inside (B = f > 0), -EDT(~B) + 0.5 outside, in lattice units (fp64); +-1 everywhere when a class is empty."""
    B = np.asarray(f) > 0
    if B.all():
        return np.ones(B.shape)
    if not B.any():
        return -np.ones(B.shape)
    return np.where(B, ndimage.distance_transform_edt(B) - 0.5, -ndimage.distance_transform_edt(~B) + 0.5)


def band(D):
    """The variables (|D| < 4), numbered in lattice order: their flat lattice indices (M,) and the neighbour table (M, 6) in the order
    -i, +i, -j, +j, -k, +k, with -1 for a neighbour outside the lattice or the band."""
    n = D.shape[0]
    pos = np.flatnonzero(np.abs(D) < BAND_RADIUS)
    index = np.full(D.size, -1, np.int64)
    index[pos] = np.arange(pos.size)
    coords = np.unravel_index(pos, D.shape)
    nb = np.full((pos.size, 6), -1, np.int64)
    for a, stride in enumerate((n * n, n, 1)):
        for s, step in enumerate((-1, 1)):
            ok = (coords[a] + step >= 0) & (coords[a] + step < n)
            nb[ok, 2 * a + s] = index[pos[ok] + step * stride]
    return pos, nb


def q_matrix(nb):
    """Q (3M, M): row 3c + a is q_a(c) = (m_a(c) - 2) x_c + the counted neighbours of c along a; m_a(c) = neighbours that do not count."""
    M = nb.shape[0]
    rows, cols, vals = [], [], []
    c = np.arange(M)
    for a in range(3):
        pair = nb[:, 2 * a:2 * a + 2]
        rows.append(3 * c + a)
        cols.append(c)
        vals.append(((pair < 0).sum(1) - 2).astype(np.float64))
        for s in range(2):
            ok = pair[:, s] >= 0
            rows.append(3 * c[ok] + a)
            cols.append(pair[ok, s])
            vals.append(np.ones(ok.sum()))
    return sparse.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * M, M))


def diag_a(nb):
    """diag(Q^T Q)_c = sum_a (m_a - 2)^2 + 2 - m_a."""
    m = np.stack([(nb[:, 2 * a:2 * a + 2] < 0).sum(1) for a in range(3)], 1)
    return ((m - 2) ** 2 + 2 - m).sum(1).astype(np.float64)


def bounds(x0):
    upper = np.where(x0 < 0, x0, np.inf)
    lower = np.where(x0 > 0, x0, -np.inf)
    upper[np.abs(upper) < 1] = 0
    lower[np.abs(lower) < 1] = 0
    return lower, upper


def energy(Q, x):
    return 0.5 * np.sum((Q @ x) ** 2)


def constrained(f, max_iters=MAX_ITERS):
    """-> (fp32 field, iterations run, band variables)"""
    D = signed_distance(f)
    B = np.asarray(f) > 0
    if B.all() or not B.any():
        return D.astype(np.float32), 0, 0
    pos, nb = band(D)
    x0 = D.ravel()[pos]
    Q = q_matrix(nb)
    A = (Q.T @ Q).tocsr()
    d = diag_a(nb)
    lower, upper = bounds(x0)
    x = x0.copy()
    live = d > 0                                   # a variable with no counted neighbour keeps x0
    e_prev = energy(Q, x0)
    it = 0
    with np.errstate(divide="ignore", invalid="ignore"):
        for t in range(1, max_iters + 1):
            it = t
            xh = -(A @ x - d * x) / d
            x = np.where(live, np.clip(0.5 * xh + 0.5 * x, lower, upper), x)
            if t % CHECK_EVERY == 0:
                e = energy(Q, x)
                if (e_prev - e) / e_prev < STOP_RATIO:
                    break
                e_prev = e
    out = D.ravel().copy()
    out[pos] = x
    return out.reshape(D.shape).astype(np.float32), it, pos.size


def gaussian(f):
    return ndimage.gaussian_filter(np.asarray(f).astype(np.float64) - 0.5, 3).astype(np.float32)


def smooth(f, method="auto", max_iters=MAX_ITERS):
    """-> (fp32 field, {"method", "iterations", "band_variables"}), as jnerf_b200.ops.mesh_smooth returns it."""
    m = pick_method(np.asarray(f).shape[0], method)
    if m == "gaussian":
        return gaussian(f), dict(method=m, iterations=0, band_variables=0)
    out, it, M = constrained(f, max_iters)
    return out, dict(method=m, iterations=it, band_variables=M)
