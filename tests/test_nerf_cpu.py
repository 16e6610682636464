"""Vanilla NeRF host logic without a GPU: FrequencyEncoder against a numpy restatement of freq_encoder.py, nerf_cfg against
projects/nerf/configs/nerf_base.py, the flat parameter layout against the reference's parameter names, and the kernels of
csrc/nerf_mlp.cu compiled for sm_90a without local-memory spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _reference_tree():
    """$NGP_REF, else the default oracle/Makefile builds the reference sources from."""
    if os.environ.get("NGP_REF"):
        return os.environ["NGP_REF"]
    m = re.search(r"^NGP_REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M)
    return m.group(1) if m else ""


def _cfg(fp16):
    from jnerf_b200.utils.config import get_cfg, update_cfg
    get_cfg().clear()
    update_cfg(fp16=fp16)


@pytest.mark.parametrize("multires,width", [(10, 63), (4, 27)])
@pytest.mark.parametrize("fp16", [True, False])
def test_frequency_encoder_matches_numpy(multires, width, fp16):
    _cfg(fp16)
    from jnerf_b200.plugin.nerf import FrequencyEncoder
    enc = FrequencyEncoder(multires)
    assert enc.out_dim == width
    x = np.random.default_rng(0).uniform(0, 1, (257, 3)).astype(np.float32)
    got = enc(torch.from_numpy(x)).numpy()
    cols = [x]
    for k in range(multires):                       # x 2^k is exact in fp32; sin / cos in fp32
        cols += [np.sin(x * np.float32(2.0 ** k)), np.cos(x * np.float32(2.0 ** k))]
    ref = np.concatenate(cols, -1)
    assert got.shape == (257, width) and got.dtype == (np.float16 if fp16 else np.float32)
    if fp16:
        # one rounding of the fp32 value: within half an fp16 ulp of it, so at most one ulp from numpy's rounding of its own value
        assert np.abs(got.astype(np.float32) - ref).max() <= 2.0 ** -11
    else:
        assert np.abs(got - ref).max() <= 1e-6


def test_nerf_cfg_is_nerf_base_key_for_key():
    ref_cfg = os.path.join(_reference_tree(), "projects", "nerf", "configs", "nerf_base.py")
    if not os.path.exists(ref_cfg):
        pytest.skip("reference tree not present")
    from jnerf_b200.runner import nerf_cfg
    ns = {}
    exec(open(ref_cfg).read(), ns)
    ref = {k: v for k, v in ns.items() if not k.startswith("__")}
    assert nerf_cfg(synthetic=False) == ref


def test_flat_layout_and_reference_names():
    from jnerf_b200.plugin import nerf
    assert nerf.N_PARAMS == 602528                  # static_assert of csrc/nerf_mlp.cu
    g = torch.Generator().manual_seed(0)
    ref = {}
    for name, ((o, i), _, _, _) in nerf.REF_LAYERS.items():
        ref[name] = ((torch.rand((o, i), generator=g) - 0.5).half().float(), (torch.rand(o, generator=g) - 0.5).half().float())
    flat = nerf.pack(ref)
    back = nerf.unpack(flat)
    for name, (W, b) in ref.items():
        assert torch.equal(back[name][0], W) and torch.equal(back[name][1], b)
    # every entry of the flat vector belongs to a reference parameter or is zero padding
    n_ref = sum(W.numel() + b.numel() for W, b in ref.values())
    assert int((flat != 0).sum()) <= n_ref and abs(float(flat.float().abs().sum()) - sum(float(W.abs().sum() + b.abs().sum()) for W, b in ref.values())) < 1e-2
    # pts_linears.5 reads concat([enc_pos (63), h4 (256)]): kernel column 63 is padding
    W5 = flat[nerf.W_OFF[5]:nerf.W_OFF[5] + 256 * 320].view(256, 320)
    assert not W5[:, 63].any() and torch.equal(W5[:, 64:].float(), ref["pts_linears.5"][0][:, 63:])


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-I",
                        os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", os.path.join(ROOT, "jnerf_b200", "csrc", "nerf_mlp.cu"), "-o",
                        str(tmp_path / "nerf_mlp.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 6 and len(spills) == 6, r.stderr[-3000:]
    assert all(int(a) == 0 and int(b) == 0 for a, b in spills), r.stderr[-3000:]


def test_runner_steps_through_the_nerf_host_glue(monkeypatch, tmp_path):
    """A few Runner steps of OriginNeRFNetworks (fp16) with the operators swapped for the fp32 torch chain (tests/nerf_cpu_backend.py):
    the occupancy update evaluates model.density, the autograd step runs nerf_fwd / nerf_bwd and one Adam+EMA sweep over the flat
    vector, the .pt checkpoint round-trips and the .pkl format is refused."""
    import nerf_cpu_backend
    import oracle_lib as ol
    fake = nerf_cpu_backend.install(monkeypatch)
    from jnerf_b200 import plugin  # noqa: F401
    from jnerf_b200 import runner as R
    from jnerf_b200.plugin import nerf
    from jnerf_b200.utils.config import get_cfg, update_cfg

    def make(seed):
        get_cfg().clear()
        update_cfg(**R.nerf_cfg(fp16=True, synthetic=True, seed=seed, n_rays_per_batch=32, target_batch_size=4096))
        cfg = get_cfg()
        cfg.dataset.train.n_images = 4
        cfg.dataset.train.H = cfg.dataset.train.W = 24
        cfg.dataset.val = None
        return R.Runner()

    r = make(1)
    m, s = r.model, r.sampler
    assert not r.fast and r._can_infer and m.params.dtype == torch.float16 and m.params.numel() == nerf.N_PARAMS
    # the occupancy update through model.density (a small sample count instead of the 2 M of a real update)
    r.cfg.m_training_step = 1
    fake.calls.clear()
    s.update_density_grid_nerf(0.95, 4096, 0)
    assert fake.calls.count("nerf_density") == 1 and bool(s.density_grid.any())
    bits, _ = ol.sphere_bitfield(0.35, cascades=s.NERF_CASCADES)
    s.density_grid_bitfield.copy_(torch.from_numpy(bits[:s.density_grid_bitfield.numel()]))
    p0 = m.params.detach().clone()
    fake.calls.clear()
    losses = [float(r.train_step_autograd().detach().mean()) for _ in range(2)]
    assert all(np.isfinite(losses))
    assert fake.calls.count("nerf_fwd") == 2 and fake.calls.count("nerf_bwd") == 2 and fake.calls.count("adam_ema") == 2
    assert not torch.equal(m.params.detach(), p0) and m.params.grad is None
    st = r.optimizer._nested_optimizer.state[0]
    assert st.p is m.params and bool(st.m.any())
    # padding of the flat vector stays zero through the optimizer
    padding = torch.ones(nerf.N_PARAMS, dtype=torch.bool)
    for name in nerf.REF_LAYERS:
        Wk, bk, cols = nerf._kernel_views(padding, name)
        for _, kc, n in cols:
            Wk[:, kc:kc + n] = False
        bk[:] = False
    assert not m.params.detach()[padding].any()
    # .pt round trip; .pkl is the NGP parameter layout only
    path = str(tmp_path / "nerf.pt")
    r.save_ckpt(path)
    r2 = make(2)
    assert not torch.equal(r2.model.params.detach(), m.params.detach())
    r2.load_ckpt(path)
    assert torch.equal(r2.model.params.detach(), m.params.detach()) and r2.cfg.m_training_step == r.cfg.m_training_step
    assert torch.equal(r2.optimizer._nested_optimizer.state[0].m, st.m)
    with pytest.raises(NotImplementedError):
        r.save_ckpt(str(tmp_path / "nerf.pkl"))
    with pytest.raises(NotImplementedError):
        r.extract_mesh(str(tmp_path / "mesh"), resolution=8)
