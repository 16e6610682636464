"""Mesh extraction and params.pkl for vanilla NeRF (OriginNeRFNetworks, fp16 kernels) on the H100: the density lattice of
csrc/nerf_lattice.cu against ngp_nerf_density bit for bit and against the float64 chain of tests/nerf_mlp_ref.py, NerfRunner.extract_mesh end
to end on a briefly trained lego stand-in (closed mesh, vertex colours replayed through march -> nerf_fwd -> composite_infer,
reproducible files, --mcube_smooth), a .pkl resume that trains on bit for bit like a .pt resume, and a reference-style file without the
fp32 optimizer copies that renders what its source renders -- all through NerfRunner."""
import os

import numpy as np
import pytest
import torch

import mesh_oracle as mo
import nerf_mlp_ref as R
from test_mesh_cpu import assert_closed_oriented
from test_nerf_gpu import LR, _setup

pytestmark = pytest.mark.gpu


def npy(t):
    return t.detach().cpu().numpy()


def spanning_params(ops, nerf, P):
    """P with alpha_linear rescaled so that alpha over the unit cube spans several integers, about half of it positive."""
    ref = nerf.unpack(P)
    a0 = ops.nerf_density(torch.from_numpy(mo.lattice_positions(24)).cuda(), P).float()
    k = 4.0 / float(a0.std())
    W, b = ref["alpha_linear"]
    ref["alpha_linear"] = (W * k, (b - a0.median()) * k + 1.5)
    return nerf.pack(ref)


@pytest.mark.parametrize("n", [64, 37])                                  # 37^3 rows: the last tile is partial
def test_lattice_is_the_density_kernel_bit_for_bit(n):
    from jnerf_b200 import ops
    nerf, P = _setup(seed=2)
    P = spanning_params(ops, nerf, P)
    field = ops.nerf_density_lattice(n, P)
    assert field.shape == (n, n, n) and field.dtype == torch.float32
    alpha = ops.nerf_density(torch.from_numpy(mo.lattice_positions(n)).cuda(), P).float()
    assert torch.equal(field.reshape(-1), torch.trunc(torch.clamp_min(alpha, 0)))
    assert len(torch.unique(field)) >= 4                                  # the field spans several integers


def test_lattice_against_the_float64_chain():
    """Every entry is the truncation of the exact (float64) alpha, except where that alpha lies within the per-entry bound of an
    integer step (1, 2, ...): there the two may differ by one.  The bound is 4 2^-11 (1 + the sum of magnitudes of alpha_linear's
    terms): eleven fp16 roundings and the encoding's, each at most 2^-12 relative, through layers of near-unit gain.  On an H100 the
    kernel's alpha came within a tenth of it (the largest ratio is printed)."""
    from jnerf_b200 import ops
    nerf, P = _setup(seed=3)
    P = spanning_params(ops, nerf, P)
    n = 48
    field = ops.nerf_density_lattice(n, P).reshape(-1).double()
    x = torch.from_numpy(mo.lattice_positions(n)).cuda()
    enc, _ = R.freq_encoding(x, 10)
    sv, out = R.forward_chain(P, enc, torch.zeros((x.shape[0], 32), dtype=torch.float64, device="cuda"))
    a64 = out[:, 3]
    W8, b8 = R.layer_params(P, 8)
    mag = R.layer_input(sv, 8).abs() @ W8[0].abs() + b8[0].abs()
    bound = 4 * 2.0 ** -11 * (1 + mag)
    want = torch.trunc(torch.clamp_min(a64, 0))
    near = ((a64 - torch.round(a64)).abs() <= bound) & (torch.round(a64) >= 1)
    print(f"[nerf-lattice] n={n}: entries near an integer step {int(near.sum())} of {near.numel()}, "
          f"largest |alpha - alpha64| / bound over all entries "
          f"{float(((ops.nerf_density(x, P).double() - a64).abs() / bound).max()):.3f}")
    assert torch.equal(field[~near], want[~near])
    assert float((field - want).abs().max()) <= 1
    assert float(near.double().mean()) < 0.2 and len(torch.unique(field)) >= 4


# ---------------------------------------------------------------------------------------------------------------- end to end
def _fresh(seed):
    """A NerfRunner of nerf_cfg on the 96x96 lego stand-in at test_nerf_gpu.py's learning rate."""
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200.nerf_runner import NerfRunner
    from jnerf_b200.runner import nerf_cfg
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(**nerf_cfg(fp16=True, synthetic=True, seed=seed, optim=dict(type="Adam", lr=LR, eps=1e-15, betas=(0.9, 0.99))))
    cfg = get_cfg()
    cfg.dataset.train.n_images = 8
    cfg.dataset.train.H = cfg.dataset.train.W = 96
    cfg.dataset.val = None
    return NerfRunner()


@pytest.fixture(scope="module")
def trained():
    r = _fresh(7)
    r.train(400)
    torch.cuda.synchronize()
    return r


def test_extract_mesh_end_to_end(trained, tmp_path):
    from jnerf_b200 import ops
    r = trained
    s, m = r.sampler, r.model
    rng0 = s.rng.copy()
    res = r.extract_mesh(str(tmp_path / "a"), resolution=128)
    print(f"[nerf-mesh] 128^3: {res['n_verts_origin']} / {res['n_tris_origin']} -> {res['n_verts']} / {res['n_tris']} vertices / triangles, "
          f"stage ms {res['stage_ms']}")
    assert res["n_tris"] > 1000 and res["n_verts"] > 500 and res["n_tris"] <= res["n_tris_origin"]
    assert_closed_oriented(res["triangles"])
    # the colours: the same rays and RNG state through march -> nerf_fwd -> composite_infer, batch by batch
    tile = r.cfg.n_rays_per_batch
    rng = rng0.copy()
    o, d = torch.from_numpy(res["origins"]).cuda(), torch.from_numpy(res["dirs"]).cuda()
    rgb, alpha = [], []
    for p in range(0, o.shape[0], tile):
        coords, _, numsteps, counters = ops.march(o[p:p + tile].contiguous(), d[p:p + tile].contiguous(), s.density_grid_bitfield, s.aabb_range,
                                                  s.max_samples, s.cone_angle_constant, s.near_distance, s.NERF_CASCADES, s.const_dt, rng)
        ops.pcg32_advance(rng)
        out, _ = ops.nerf_fwd(coords, m.params, n_dev=counters[1:2])
        c, a = ops.composite_infer(out, coords, numsteps, s.NERF_CASCADES)
        rgb.append(npy(c))
        alpha.append(npy(a))
    assert np.array_equal(s.rng, rng)
    img = np.concatenate(rgb).astype(np.float64) + np.asarray(r.background_color, np.float64) * (1 - np.concatenate(alpha).astype(np.float64))
    assert np.array_equal((img * 255 + 0.5).clip(0, 255).astype(np.uint8), res["colors"])
    assert res["colors"].std() > 0
    vm = res["vertices"][:, [1, 0, 2]]
    assert np.allclose(res["origins"] + 0.2 * res["dirs"], vm, atol=1e-6)
    # two runs from the same RNG state write byte-identical files
    s.rng[:] = rng0
    r.extract_mesh(str(tmp_path / "b"), resolution=128)
    for f in ("mesh-origin.ply", "mesh-color.ply"):
        assert open(tmp_path / "a" / f, "rb").read() == open(tmp_path / "b" / f, "rb").read(), f
    assert os.path.getsize(tmp_path / "a" / "mesh-color.ply") > 0
    # the smoothed lattice, marched at 0
    sm = r.extract_mesh(str(tmp_path / "c"), resolution=128, mcube_smooth=True)
    assert list(sm["stage_ms"])[:3] == ["density_lattice", "smooth", "marching_cubes"] and sm["n_tris"] > 1000


# ---------------------------------------------------------------------------------------------------------------- params.pkl
def test_pkl_resume_trains_on_like_a_pt_resume(trained, tmp_path):
    r = trained
    step0 = r.cfg.m_training_step
    pt, pkl = str(tmp_path / "ckpt.pt"), str(tmp_path / "params.pkl")
    r.save_ckpt(pt)
    r.save_ckpt(pkl)
    got = []
    for path in (pkl, pt):                                                # one after the other: the configuration is global
        x = _fresh(11)
        x.load_ckpt(path)
        assert x.cfg.m_training_step == step0 and torch.equal(x.model.params, r.model.params)
        x.train(24)
        assert x.cfg.m_training_step == step0 + 24
        st = x.optimizer._nested_optimizer.state[0]
        got.append([t.detach().clone() for t in (x.model.params, st.m, st.v, st.master)])
        del x
    assert all(torch.equal(a, b) for a, b in zip(*got)) and not torch.equal(got[0][0], r.model.params)


def test_reference_style_pkl_renders_the_source_view(trained, tmp_path):
    from jnerf_b200.utils import ckpt_compat as cc
    r = trained
    path = str(tmp_path / "params.pkl")
    r.save_ckpt(path)
    ref = cc.read_reference_ckpt(path)
    for pg in (ref["nested_optimizer"]["defaults"]["param_groups"][0], ref["ema_optimizer"]["defaults"]["param_groups"][0]):
        for k in [k for k in pg if k.endswith("_f32")]:
            del pg[k]
    stripped = str(tmp_path / "stripped.pkl")
    cc.write_reference_ckpt(ref, stripped)
    c = _fresh(12)
    c.load_ckpt(stripped)
    assert torch.equal(c.model.params, r.model.params)
    assert torch.isfinite(c.optimizer._nested_optimizer.state[0].v).all()
    rng0 = r.sampler.rng.copy()
    img_r, _ = r.render_img_nosync("train", 1)
    c.sampler.rng[:] = rng0
    img_c, _ = c.render_img_nosync("train", 1)
    assert torch.equal(img_r, img_c)
