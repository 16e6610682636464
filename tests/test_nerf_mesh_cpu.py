"""Mesh extraction and the reference's params.pkl for vanilla NeRF (OriginNeRFNetworks, NerfRunner) without a GPU: the host glue with the
operators swapped for the fp32 torch chain (tests/nerf_cpu_backend.py) and the mesh oracle (tests/mesh_cpu_backend.py), the C ABI's
resolution check of ngp_nerf_density_lattice, and utils/ckpt_compat.py's by-name mapping of the 24 reference tensors in both modes."""
import numpy as np
import pytest
import torch

import mesh_cpu_backend
import mesh_oracle as mo
import nerf_cpu_backend
import oracle_lib as ol
from test_ckpt_compat import reference_style_ckpt
from test_mesh_cpu import assert_closed_oriented, read_ply

from jnerf_b200.utils import ckpt_compat as cc


def make_nerf_runner(seed, fp16=True):
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.nerf_runner import NerfRunner
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**R.nerf_cfg(fp16=fp16, synthetic=True, seed=seed, n_rays_per_batch=32, target_batch_size=4096))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 4
    cfg.dataset.train.H = cfg.dataset.train.W = 24
    cfg.dataset.val = None
    return NerfRunner()


def test_nerf_runner_round_trips_pkl_and_refuses_other_models(monkeypatch, tmp_path):
    """Two autograd steps of NerfRunner (fp16) on the fp32 torch chain (tests/nerf_cpu_backend.py), then the reference's .pkl written
    and read back into a runner of another seed: parameters, the fp32 optimizer state, counters and the sampler state, exactly."""
    nerf_cpu_backend.install(monkeypatch)
    r = make_nerf_runner(1)
    s = r.sampler
    bits, _ = ol.sphere_bitfield(0.35, cascades=s.NERF_CASCADES)
    s.density_grid_bitfield.copy_(torch.from_numpy(bits[:s.density_grid_bitfield.numel()]))
    r.cfg.m_training_step = 1
    for _ in range(2):
        r.train_step_autograd()
    st = r.optimizer._nested_optimizer.state[0]
    assert bool(st.m.any())
    path = str(tmp_path / "params.pkl")
    r.save_ckpt(path)
    assert list(cc.read_reference_ckpt(path)["model"]) == KEYS
    r2 = make_nerf_runner(2)
    assert not torch.equal(r2.model.params.detach(), r.model.params.detach())
    r2.load_ckpt(path)
    assert torch.equal(r2.model.params.detach(), r.model.params.detach()) and r2.cfg.m_training_step == 3
    st2 = r2.optimizer._nested_optimizer.state[0]
    assert torch.equal(st2.m, st.m) and torch.equal(st2.v, st.v) and torch.equal(st2.master, st.master)
    assert r2.optimizer._nested_optimizer.n_step == 2 and r2.ema_optimizer.steps == 2 and r2.optimizer.steps == r.optimizer.steps
    assert torch.equal(r2.sampler.density_grid, s.density_grid) and torch.equal(r2.sampler.density_grid_bitfield, s.density_grid_bitfield)
    assert np.array_equal(r2.sampler.rng, s.rng)
    # an NGP config is Runner's
    from jnerf_b200 import runner as R
    from jnerf_b200.nerf_runner import NerfRunner
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**R.lego_cfg(fp16=True, synthetic=True, seed=1, n_rays_per_batch=32, target_batch_size=4096))
    get_cfg().dataset.train.n_images, get_cfg().dataset.train.H, get_cfg().dataset.train.W = 2, 8, 8
    get_cfg().dataset.val = None
    with pytest.raises(ValueError, match="use Runner"):
        NerfRunner()


# ---- NerfRunner.extract_mesh ------------------------------------------------------------------------------------------------------
def plant_octahedron(params):
    """Weights of the flat fp16 vector whose alpha is 4 - 12 (|x - .5| + |y - .5| + |z - .5|): pts_linears.0 makes relu(+-(x_d - .5)) in
    units 0..5, pts_linears.1..7 pass them on, alpha_linear sums them.  The solid is inside the unit cube, away from its faces."""
    from jnerf_b200.plugin import nerf
    ref = nerf.unpack(params.detach())
    for name in [f"pts_linears.{i}" for i in range(8)] + ["alpha_linear"]:
        ref[name][0].zero_()
        ref[name][1].zero_()
    W0, b0 = ref["pts_linears.0"]
    for d in range(3):                                                 # encoding column d is x_d itself
        W0[2 * d, d], b0[2 * d] = 1.0, -0.5
        W0[2 * d + 1, d], b0[2 * d + 1] = -1.0, 0.5
    for i in range(1, 8):
        W, _ = ref[f"pts_linears.{i}"]
        c0 = 63 if i == 5 else 0                                       # pts_linears.5 reads concat([enc, h4])
        for u in range(6):
            W[u, c0 + u] = 1.0
    ref["alpha_linear"][0][0, :6] = -12.0
    ref["alpha_linear"][1][0] = 4.0
    with torch.no_grad():
        params.copy_(nerf.pack(ref))


def chain_lattice(fake, n, params):
    """ops.nerf_density_lattice restated: the fp32 chain of tests/nerf_cpu_backend.py on mesh_oracle.lattice_positions, rounded to
    fp16 as the kernel's alpha is, then float(int(max(alpha, 0)))."""
    fake._log("nerf_density_lattice")
    if not 2 <= int(n) <= 1024:
        raise RuntimeError(f"nerf_density_lattice: resolution {n} is outside [2, 1024]")
    alpha = nerf_cpu_backend._chain(params, torch.from_numpy(mo.lattice_positions(n))).half().float()
    return torch.trunc(torch.clamp_min(alpha, 0)).reshape(n, n, n)


def test_nerf_runner_extract_mesh_on_cpu(monkeypatch, tmp_path):
    fake = nerf_cpu_backend.install(monkeypatch)
    mesh_cpu_backend.install(monkeypatch, fake)
    from jnerf_b200 import ops
    r = make_nerf_runner(3)
    s = r.sampler
    bits, _ = ol.sphere_bitfield(0.35, cascades=s.NERF_CASCADES)
    s.density_grid_bitfield.copy_(torch.from_numpy(bits[:s.density_grid_bitfield.numel()]))
    plant_octahedron(r.model.params)
    monkeypatch.setattr(ops, "nerf_density_lattice", lambda n, params: chain_lattice(fake, n, params))
    marched = []
    march = ops.march

    def spy(rays_o, rays_d, *a, **k):
        marched.append((rays_o.clone().numpy(), rays_d.clone().numpy()))
        return march(rays_o, rays_d, *a, **k)
    monkeypatch.setattr(ops, "march", spy)
    n = 20
    rng0 = s.rng.copy()
    fake.calls.clear()
    res = r.extract_mesh(str(tmp_path), resolution=n)
    nb = -(-res["n_verts"] // 32)
    assert fake.calls == ["nerf_density_lattice", "marching_cubes", "mesh_largest_component", "mesh_vertex_normals"] + \
        ["march", "nerf_fwd", "composite_infer"] * nb
    assert list(res["stage_ms"]) == ["density_lattice", "marching_cubes", "write_origin", "component_normals", "colour"]
    rng = rng0.copy()
    for _ in range(nb):
        rng = ol.pcg32_advance(rng)
    assert np.array_equal(s.rng, rng)                                   # one advance per batch
    # the octahedron: a closed, oriented surface, symmetric about the centre
    assert res["n_tris"] > 100 and res["n_tris"] == res["n_tris_origin"]
    assert_closed_oriented(res["triangles"])
    c = (n - 1) / (2 * n)                                               # the lattice centre in the /N vertex frame
    assert np.allclose(res["vertices"].mean(0), c, atol=1e-5)
    # the files carry the result
    vp, v0, f0 = read_ply(tmp_path / "mesh-origin.ply")
    assert len(v0) == res["n_verts_origin"] and len(f0) == res["n_tris_origin"]
    vp, v1, f1 = read_ply(tmp_path / "mesh-color.ply")
    assert np.array_equal(np.stack([v1["x"], v1["y"], v1["z"]], 1), res["vertices"]) and np.array_equal(f1, res["triangles"])
    assert np.array_equal(np.stack([v1["red"], v1["green"], v1["blue"]], 1), res["colors"])
    # colour rays: from 0.2 outside the vertex along the unit normal, towards the centre
    o = np.concatenate([mm[0] for mm in marched])
    d = np.concatenate([mm[1] for mm in marched])
    vm = res["vertices"][:, [1, 0, 2]]
    assert np.allclose(o + 0.2 * d, vm, atol=1e-6) and np.allclose(np.linalg.norm(d, axis=1), 1, atol=1e-5)
    assert (np.einsum("ij,ij->i", c - vm, d) > 0).all()


def test_extract_mesh_refuses_the_fp32_nerf_chain(monkeypatch, tmp_path):
    nerf_cpu_backend.install(monkeypatch)
    r = make_nerf_runner(4, fp16=False)
    with pytest.raises(NotImplementedError, match="fp16=True"):
        r.extract_mesh(str(tmp_path / "never-created"), resolution=8)
    path = str(tmp_path / "params.pkl")                                # .pkl works in this mode too
    r.save_ckpt(path)
    r.load_ckpt(path)
    with pytest.raises(NotImplementedError, match="fp16=True"):
        r.model.density_lattice(8)
    assert not (tmp_path / "never-created").exists()


def test_c_abi_rejects_bad_resolutions():
    from jnerf_b200 import build, lib as L
    build.build()
    lib = L.load()
    for n in (0, 1, 1025):
        assert lib.ngp_nerf_density_lattice(None, n, None, None) != 0
        assert b"[2, 1024]" in lib.ngp_last_error()


# ---- params.pkl of OriginNeRFNetworks ---------------------------------------------------------------------------------------------
KEYS = [f"{n}.{p}" for n in [f"pts_linears.{i}" for i in range(8)] + ["views_linears.0", "feature_linear", "alpha_linear", "rgb_linear"]
        for p in ("weight", "bias")]


def ref_tensors(seed, scale=1.0):
    """{reference key: fp32 array} of the reference shapes."""
    rng = np.random.default_rng(seed)
    return {k: (rng.standard_normal(shp) * scale).astype(np.float32) for k, shp in cc.nerf_reference_shapes().items()}


def native_ckpt(fp16, seed=0):
    """The dict Runner.save_ckpt builds for OriginNeRFNetworks, in either mode."""
    from jnerf_b200.plugin import nerf
    p, m, v = ref_tensors(seed, 0.1), ref_tensors(seed + 1, 1e-3), {k: np.abs(t) for k, t in ref_tensors(seed + 2, 1e-6).items()}
    master = {k: t + np.float32(1e-4) for k, t in p.items()}

    def join(t, dtype):
        return nerf.pack({n: (torch.from_numpy(t[f"{n}.weight"]), torch.from_numpy(t[f"{n}.bias"])) for n in nerf.REF_ORDER}, dtype=dtype)
    if fp16:
        model = {"params": join(p, torch.float16)}
        lists = {k: [join(t, torch.float32)] for k, t in (("m", m), ("v", v), ("master", master))}
    else:
        model = {k: torch.from_numpy(p[k]) for k in KEYS}
        lists = {k: [torch.from_numpy(t[key].reshape(-1)) for key in KEYS] for k, t in (("m", m), ("v", v), ("master", master))}
    G = 128 ** 3
    rng = np.random.default_rng(seed + 3)
    sampler = {"density_grid": torch.from_numpy(rng.random(G, dtype=np.float32)),
               "density_grid_bitfield": torch.from_numpy(rng.integers(0, 256, G // 8, dtype=np.uint8)),
               "density_grid_mean": torch.tensor([0.25]), "density_grid_ema_step": torch.tensor([40], dtype=torch.int32),
               "n_rays_per_batch": 512, "rng": torch.tensor([987654321, 5])}
    return {"global_step": 640, "model": model, "sampler": sampler, "optimizer": {"steps": 640, "m_learning_rate_factor": 1},
            "nested_optimizer": dict(n_step=640, lr=5e-4, **lists), "ema_optimizer": {"steps": 640, "decay": 0.95}}


def to_numpy(x):
    return cc._to_numpy(x)


def assert_same_native(a, b):
    a, b = to_numpy(a), to_numpy(b)
    assert list(a["model"]) == list(b["model"])
    for k in a["model"]:
        assert a["model"][k].dtype == b["model"][k].dtype and np.array_equal(a["model"][k].reshape(-1), b["model"][k].reshape(-1)), k
    for k in ("m", "v", "master"):
        assert len(a["nested_optimizer"][k]) == len(b["nested_optimizer"][k])
        for x, y in zip(a["nested_optimizer"][k], b["nested_optimizer"][k]):
            assert x.dtype == y.dtype == np.float32 and np.array_equal(x.reshape(-1), y.reshape(-1)), k
    assert a["global_step"] == b["global_step"] and a["nested_optimizer"]["n_step"] == b["nested_optimizer"]["n_step"]
    assert a["ema_optimizer"]["steps"] == b["ema_optimizer"]["steps"] and a["optimizer"]["steps"] == b["optimizer"]["steps"]
    for k in ("density_grid", "density_grid_bitfield", "density_grid_mean", "density_grid_ema_step", "rng"):
        assert np.array_equal(np.asarray(a["sampler"][k]).reshape(-1), np.asarray(b["sampler"][k]).reshape(-1)), k
    assert int(a["sampler"]["n_rays_per_batch"]) == int(b["sampler"]["n_rays_per_batch"])


@pytest.mark.parametrize("fp16", [True, False])
def test_written_file_holds_the_reference_tensors(fp16, tmp_path):
    ref = cc.nerf_native_to_reference(native_ckpt(fp16), param_dtype=np.float16 if fp16 else np.float32)
    path = str(tmp_path / "params.pkl")
    cc.write_reference_ckpt(ref, path)
    ref = cc.read_reference_ckpt(path)
    dt = np.float16 if fp16 else np.float32
    assert list(ref["model"]) == KEYS and len(KEYS) == 24
    assert ref["model"]["pts_linears.5.weight"].shape == (256, 319) and ref["model"]["pts_linears.0.weight"].shape == (256, 63)
    assert ref["model"]["views_linears.0.weight"].shape == (128, 283) and ref["model"]["alpha_linear.weight"].shape == (1, 256)
    assert ref["model"]["rgb_linear.bias"].shape == (3,)
    for k, shp in cc.nerf_reference_shapes().items():
        assert ref["model"][k].shape == shp and ref["model"][k].dtype == dt, k
    pg = ref["nested_optimizer"]["defaults"]["param_groups"][0]
    ema = ref["ema_optimizer"]["defaults"]["param_groups"][0]
    for lst, want in ((pg["values"], dt), (pg["m"], dt), (ema["values"], dt), (pg["values_f32"], np.float32), (pg["m_f32"], np.float32),
                      (ema["values_f32"], np.float32)):
        assert [t.shape for t in lst] == [cc.nerf_reference_shapes()[k] for k in KEYS] and all(t.dtype == want for t in lst)
    assert ref["optimizer"]["defaults"]["steps"] == 640 and ref["ema_optimizer"]["defaults"]["steps"] == 640
    assert ref["sampler"]["density_grid_mean"].shape == (16384,) and ref["sampler"]["density_grid"].shape == (128 ** 3,)
    # the flat layout's padding is not in the file: every reference tensor is the corresponding slice of the kernels' vector
    want = ref_tensors(0, 0.1)
    for k in KEYS:
        assert np.array_equal(ref["model"][k], want[k].astype(dt)), k


@pytest.mark.parametrize("fp16", [True, False])
def test_native_pkl_native_round_trip_is_lossless(fp16, tmp_path):
    nat = native_ckpt(fp16)
    path = str(tmp_path / "params.pkl")
    cc.write_reference_ckpt(cc.nerf_native_to_reference(nat, param_dtype=np.float16 if fp16 else np.float32), path)
    back = cc.nerf_reference_to_native(cc.read_reference_ckpt(path), fp16)
    assert_same_native(nat, back)
    # padding of the flat vectors is zero
    if fp16:
        from jnerf_b200.plugin import nerf
        pad = torch.ones(nerf.N_PARAMS, dtype=torch.bool)
        for name in nerf.REF_LAYERS:
            Wk, bk, cols = nerf._kernel_views(pad, name)
            for _, kc, n in cols:
                Wk[:, kc:kc + n] = False
            bk[:] = False
        for t in [back["model"]["params"]] + back["nested_optimizer"]["m"] + back["nested_optimizer"]["master"]:
            assert not np.asarray(t)[pad.numpy()].any()


def test_a_file_of_one_mode_loads_in_the_other(tmp_path):
    from jnerf_b200.plugin import nerf
    # fp16 file -> fp32 model: the fp16 values exactly, the fp32 optimizer state exactly
    nat16 = native_ckpt(True, seed=10)
    p16 = str(tmp_path / "a.pkl")
    cc.write_reference_ckpt(cc.nerf_native_to_reference(nat16, param_dtype=np.float16), p16)
    got = cc.nerf_reference_to_native(cc.read_reference_ckpt(p16), fp16=False)
    ref16 = nerf.unpack(nat16["model"]["params"])
    m16 = nerf.unpack(nat16["nested_optimizer"]["m"][0])
    assert list(got["model"]) == KEYS
    for i, k in enumerate(KEYS):
        name, part = k.rsplit(".", 1)
        j = 0 if part == "weight" else 1
        assert np.array_equal(got["model"][k].astype(np.float32), ref16[name][j].numpy()), k
        assert np.array_equal(got["nested_optimizer"]["m"][i], m16[name][j].numpy().reshape(-1)), k
    # fp32 file -> fp16 model: the parameters rounded to fp16 once, the optimizer state in fp32
    nat32 = native_ckpt(False, seed=20)
    p32 = str(tmp_path / "b.pkl")
    cc.write_reference_ckpt(cc.nerf_native_to_reference(nat32, param_dtype=np.float32), p32)
    got = cc.nerf_reference_to_native(cc.read_reference_ckpt(p32), fp16=True)
    want = {n: (nat32["model"][f"{n}.weight"], nat32["model"][f"{n}.bias"]) for n in nerf.REF_ORDER}
    assert got["model"]["params"].dtype == np.float16
    assert np.array_equal(got["model"]["params"], nerf.pack(want).numpy())
    master = nerf.unpack(torch.from_numpy(got["nested_optimizer"]["master"][0]))
    for i, k in enumerate(KEYS):
        name, part = k.rsplit(".", 1)
        assert np.array_equal(master[name][0 if part == "weight" else 1].numpy().reshape(-1), nat32["nested_optimizer"]["master"][i].numpy()), k


def reference_written(seed=0):
    """A params.pkl as the reference writes it for nerf_base.py (fp16=True): fp16 tensors, fp16 moments, no *_f32 keys."""
    ref = reference_style_ckpt(seed=seed, extra_vars=False)
    rng = np.random.default_rng(seed + 100)
    shapes = cc.nerf_reference_shapes()
    h = lambda shp, s: (rng.standard_normal(shp) * s).astype(np.float16)          # noqa: E731
    ref["model"] = {k: h(shp, 0.1) for k, shp in shapes.items()}
    m = [h(shp, 1e-3) for shp in shapes.values()]
    v = [np.abs(h(shp, 1e-7)) for shp in shapes.values()]                      # mostly subnormal or flushed to 0 in fp16
    ref["nested_optimizer"]["defaults"]["param_groups"] = [{"values": v, "m": m}]
    ref["ema_optimizer"]["defaults"]["param_groups"] = [{"values": [t.copy() for t in ref["model"].values()]}]
    return ref


@pytest.mark.parametrize("fp16", [True, False])
def test_reference_written_file_gets_the_moment_floor(fp16):
    from jnerf_b200.plugin import nerf
    ref = reference_written(seed=4)
    nat = cc.nerf_reference_to_native(ref, fp16)
    pg = ref["nested_optimizer"]["defaults"]["param_groups"][0]
    flushed_any = False
    for i, k in enumerate(KEYS):
        m16, v16 = pg["m"][i].astype(np.float32), pg["values"][i].astype(np.float32)
        flushed = (v16 == 0) & (m16 != 0)
        flushed_any |= bool(flushed.any())
        want_v, want_m = np.where(flushed, m16 * m16, v16), m16
        if fp16:
            name, part = k.rsplit(".", 1)
            j = 0 if part == "weight" else 1
            got_v = nerf.unpack(torch.from_numpy(nat["nested_optimizer"]["v"][0]))[name][j].numpy()
            got_m = nerf.unpack(torch.from_numpy(nat["nested_optimizer"]["m"][0]))[name][j].numpy()
        else:
            got_v, got_m = nat["nested_optimizer"]["v"][i].reshape(v16.shape), nat["nested_optimizer"]["m"][i].reshape(m16.shape)
        assert np.array_equal(got_v, want_v) and np.array_equal(got_m, want_m), k
    assert flushed_any
    assert nat["nested_optimizer"]["n_step"] == nat["ema_optimizer"]["steps"] == 1234 and "n_rays_per_batch" not in nat["sampler"]


def test_mismatched_and_foreign_files_are_refused():
    ref = reference_written(seed=5)
    bad = reference_written(seed=5)
    bad["nested_optimizer"]["defaults"]["param_groups"][0]["m"][4] = np.zeros((256, 255), np.float16)   # pts_linears.2.weight
    with pytest.raises(ValueError, match="pts_linears.2.weight"):
        cc.nerf_reference_to_native(bad, True)
    bad = reference_written(seed=5)
    bad["model"]["feature_linear.weight"] = np.zeros((256, 255), np.float16)
    with pytest.raises(ValueError, match="feature_linear.weight"):
        cc.nerf_reference_to_native(bad, False)
    bad = reference_written(seed=5)
    bad["ema_optimizer"]["defaults"]["param_groups"][0]["values"].pop()
    with pytest.raises(ValueError, match="EMA"):
        cc.nerf_reference_to_native(bad, True)
    with pytest.raises(KeyError, match="not OriginNeRFNetworks"):
        cc.nerf_reference_to_native(reference_style_ckpt(seed=1), True)        # an NGP params.pkl
    assert cc.nerf_reference_to_native(ref, True)["model"]["params"].size > 0
