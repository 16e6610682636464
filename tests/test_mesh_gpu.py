"""Mesh extraction on the H100: the lattice query against ngp_density_fwd (bit for bit) and the oracle, marching cubes / component
filter / normals bit-identical to the oracle on analytic and random fields (N = 257 included), reproducible PLY files, and an end-to-end
extraction from a briefly trained lego stand-in whose vertex colours match the march / network / composite path."""
import os

import numpy as np
import pytest
import torch

import mesh_oracle as mo
import oracle_lib as ol
from test_mesh_cpu import assert_closed_oriented, random_field, sphere_field, torus_field, two_spheres

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from jnerf_b200 import ops as o
    return o


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def npy(t):
    return t.detach().cpu().numpy()


def test_density_lattice_matches_density_fwd_and_oracle(ops):
    n = 64
    cfg = ol.HashCfg(1, log2_hashmap_size=19)
    lv = ops.HashLevels(1, log2_hashmap_size=19)
    rng = np.random.default_rng(5)
    grid = rng.uniform(-1, 1, cfg.n_params).astype(np.float16)
    wd = rng.uniform(-1, 1, 3072).astype(np.float16)                                  # sigma_raw over several integers
    pos = mo.lattice_positions(n)
    field = npy(ops.density_lattice(n, cu(grid), lv, cu(wd)))
    sig = npy(ops.density_fwd(cu(pos), cu(grid), lv, cu(wd))).astype(np.float32)
    assert np.array_equal(field.reshape(-1), np.trunc(np.maximum(sig, 0)))           # same positions: bit for bit
    assert len(np.unique(field)) >= 3                                                  # the field spans several integers
    scales = np.ascontiguousarray(lv.table.cpu().numpy().view(np.float32).reshape(16, 8)[:, 0])
    ol.oracle().orc_set_level_scales(ol._ptr(scales))
    try:
        enc = ol.hash_fwd(cfg, pos, grid, acc32=True)
        ref = ol.mlp_fwd(wd, enc, 0)[0][:, 0].astype(np.float32)
    finally:
        ol.oracle().orc_set_level_scales(None)
    assert np.abs(sig - ref).max() <= 1e-2                                              # test_gpu_ops.py's density_fwd tolerance
    ref_field = np.trunc(np.maximum(ref, 0))
    far = np.abs(np.maximum(ref, 0) - np.round(np.maximum(ref, 0))) > 1e-2              # not within the tolerance of an integer step
    assert np.array_equal(field.reshape(-1)[far], ref_field[far]) and np.abs(field.reshape(-1) - ref_field).max() <= 1


@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres", "random", "sphere257"])
def test_mesh_stages_match_oracle_bit_for_bit(ops, name):
    field = {"sphere": lambda: sphere_field(96), "torus": lambda: torus_field(80), "two_spheres": lambda: two_spheres(64),
             "random": lambda: random_field(48, seed=9), "sphere257": lambda: sphere_field(257, 0.31)}[name]()
    v_ref, t_ref = mo.marching_cubes(field)
    v, t = ops.marching_cubes(cu(field), 0.5)
    assert np.array_equal(npy(v), v_ref) and np.array_equal(npy(t), t_ref)
    vk_ref, tk_ref = mo.mesh_largest_component(v_ref, t_ref)
    vk, tk = ops.mesh_largest_component(v, t)
    assert np.array_equal(npy(vk), vk_ref) and np.array_equal(npy(tk), tk_ref)
    n_ref = mo.mesh_vertex_normals(vk_ref, tk_ref)
    nrm = ops.mesh_vertex_normals(vk, tk)
    assert np.array_equal(npy(nrm), n_ref)
    if name != "random":
        assert_closed_oriented(npy(tk))


def test_bad_resolutions_are_rejected(ops):
    lv = ops.HashLevels(1, log2_hashmap_size=14)
    g = torch.zeros(lv.n_params, dtype=torch.float16, device="cuda")
    w = torch.zeros(3072, dtype=torch.float16, device="cuda")
    for n in (1, 1025):
        with pytest.raises(ops.lib.NgpError, match="1024"):
            ops.density_lattice(n, g, lv, w)
        with pytest.raises(ops.lib.NgpError, match="1024"):
            ops.lib.call("ngp_marching_cubes", None, n, g.data_ptr(), 0.5, g.data_ptr(), None, 0, None, 0, np.zeros(2, np.uint64).ctypes.data)


@pytest.fixture(scope="module")
def trained():
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.runner import Runner, lego_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**lego_cfg(fp16=True, synthetic=True, seed=3))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 16
    cfg.dataset.train.H = cfg.dataset.train.W = 160
    cfg.dataset.val = None
    r = Runner()
    for _ in range(400):
        r.train_step()
    torch.cuda.synchronize()
    return r


def test_extract_mesh_end_to_end(ops, trained, tmp_path):
    r = trained
    s, m = r.sampler, r.model
    rng0 = s.rng.copy()
    res = r.extract_mesh(str(tmp_path / "a"), resolution=128)
    assert res["n_tris"] > 1000 and res["n_verts"] > 500 and res["n_tris"] <= res["n_tris_origin"]
    assert_closed_oriented(res["triangles"])
    # the colours: the same rays and RNG state through march -> network -> composite_infer, batch by batch
    tile = r.cfg.n_rays_per_batch
    rng = rng0.copy()
    o, d = cu(res["origins"]), cu(res["dirs"])
    rgb, alpha = [], []
    for p in range(0, o.shape[0], tile):
        coords, _, numsteps, counters = ops.march(o[p:p + tile].contiguous(), d[p:p + tile].contiguous(), s.density_grid_bitfield, s.aabb_range,
                                                  s.max_samples, s.cone_angle_constant, s.near_distance, s.NERF_CASCADES, s.const_dt, rng)
        ops.pcg32_advance(rng)
        out, _ = ops.network_fwd(coords, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights,
                                 n_dev=counters[1:2], save_enc=False)
        c, a = ops.composite_infer(out, coords, numsteps, s.NERF_CASCADES)
        rgb.append(npy(c))
        alpha.append(npy(a))
    assert np.array_equal(s.rng, rng)
    img = np.concatenate(rgb).astype(np.float64) + np.asarray(r.background_color, np.float64) * (1 - np.concatenate(alpha).astype(np.float64))
    assert np.array_equal((img * 255 + 0.5).clip(0, 255).astype(np.uint8), res["colors"])
    assert res["colors"].std() > 0
    # rays: 0.2 outside the vertex, unit length, into the object
    vm = res["vertices"][:, [1, 0, 2]]
    assert np.allclose(res["origins"] + 0.2 * res["dirs"], vm, atol=1e-6)
    # two runs from the same RNG state write byte-identical files
    s.rng[:] = rng0
    r.extract_mesh(str(tmp_path / "b"), resolution=128)
    for f in ("mesh-origin.ply", "mesh-color.ply"):
        assert open(tmp_path / "a" / f, "rb").read() == open(tmp_path / "b" / f, "rb").read(), f
    assert os.path.getsize(tmp_path / "a" / "mesh-color.ply") > 0
