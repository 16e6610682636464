"""Checkpoint wire format of the reference (SURVEY.md 8f N4): `params.pkl` written by Runner.save_ckpt
(runner/runner.py:123-131) with jt.save and read back by Runner.load_ckpt (:133-151).

What the file is.  jt.save converts every jt.Var to a numpy array and pickles the nested dict; Jittor's pickle writer is outside
the reference tree (third-party, version unpinned -- SURVEY 8c), so the container is restated from its published behaviour:
pickle protocol 4, followed by the 20-byte SHA-1 of the pickle bytes and the 8-byte tag b"HCAJSLHD"; older Jittor versions
wrote the bare pickle.  `read_reference_ckpt` accepts both (and verifies the digest when the tag is present);
`write_reference_ckpt` writes the tagged form.  The STRUCTURE of the dict, on the other hand, is pinned by the reference's own
load_ckpt, which indexes it explicitly:

    {'global_step': int,
     'model':            {'pos_encoder.m_grid': (n_params,), 'density_mlp.con_weights': (3072,), 'rgb_mlp.con_weights': (7168,), ...},
     'sampler':          {'density_grid': f32[C*128^3], 'density_grid_bitfield': u8[C*128^3/8], 'density_grid_mean': f32[16384],
                          'density_grid_ema_step': i32[1], ...},
     'optimizer':        {'defaults': {'steps', 'm_learning_rate_factor', 'base_lr', 'decay_*'}},            # ExpDecay, expdecay.py:8-19
     'nested_optimizer': {'defaults': {'lr', 'eps', 'betas', 'param_groups': [{'values': [v_i], 'm': [m_i], ...}]}},   # jt.nn.Adam: values = 2nd moment
     'ema_optimizer':    {'defaults': {'decay', 'steps', 'param_groups': [{'values': [ema_i]}]}}}             # ema.py:9-24

Parameters are matched by element count, not by key or position: whether Jittor also sweeps the Vars held by jt.Function members
(GridEncode's scratch buffers) into state_dict()/parameters() cannot be checked without Jittor (SURVEY 8c), and the three
trainable tensors of NGP have distinct sizes.  `nn.Linear` checkpoints (the reference's fp32 fallback, ngp_network.py:59-67) are
folded into the flat `con_weights` layout of OPS/fully_fused_mlp.py:26-40.

Vanilla NeRF (OriginNeRFNetworks, projects/nerf/configs/nerf_base.py) is matched by NAME instead: most of its 24 tensors are
(256, 256), so element counts cannot tell them apart.  Its model dict holds pts_linears.{0..7}, views_linears.0, feature_linear,
alpha_linear and rgb_linear, each .weight (out, in) and .bias, and the i-th entry of the Adam / EMA lists belongs to the i-th key of
that dict (Jittor's state_dict() and parameters() traverse the modules in the same order).  Every entry's shape is checked against its
key's; but a file whose lists swapped two equal-shaped tensors passes every check and loads them crossed, which cannot be detected
without Jittor (SURVEY 8c).  Either native form maps to the same file: the fp16 kernels' flat vector through plugin/nerf.py's
pack / unpack (padding zero), the fp32 nn.Linear chain one to one.

Two reference behaviours that are NOT reproduced (documented deviations):
  * the reference excludes Adam's `n_step` from its state (optims/adam.py:13-16), so its bias correction restarts at 1 after a
    resume; here n_step is restored from the EMA step counter (the two advance together, runner.py:75-76);
  * `n_rays_per_batch` and the pcg32 state are not Vars and are therefore not in the reference file; they are carried under
    extra keys ('sampler' -> 'n_rays_per_batch', 'rng') which the reference's load_state_dict ignores.
  * Adam moments and EMA values are written in the PARAMETER dtype (fp16 for the NGP configs with fp16=True), as jt.nn.Adam / EMA
    allocate them (`jt.zeros(p.shape, p.dtype)`, `p.copy()`): a .pkl round trip rounds this repo's fp32 optimizer state to fp16.
    Use the native `.pt` format for a lossless resume; `.pkl` is the interchange format with the reference.
All functions work on numpy arrays / python scalars; nothing here touches the GPU."""
import hashlib
import io
import pickle

import numpy as np

_TAG = b"HCAJSLHD"
N_DENSITY, N_RGB = 3072, 7168                 # 32*64 + 64*16 ; 32*64 + 64*64 + 64*16  (ngp_network.py:52-53)


class _NumpyOnlyUnpickler(pickle.Unpickler):
    """A checkpoint is data: only numpy array reconstruction and builtin containers are allowed to be unpickled."""
    _OK = {("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "_reconstruct"), ("numpy", "ndarray"), ("numpy", "dtype"),
           ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar"), ("collections", "OrderedDict"),
           ("numpy.core.numeric", "_frombuffer"), ("numpy._core.numeric", "_frombuffer")}

    def find_class(self, module, name):
        if (module, name) in self._OK:
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"params.pkl may only contain numpy arrays and builtin containers, found {module}.{name}")


def read_reference_ckpt(path):
    raw = open(path, "rb").read()
    if raw.endswith(_TAG):
        body, digest = raw[:-28], raw[-28:-8]
        if hashlib.sha1(body).digest() != digest:
            raise ValueError(f"{path}: SHA-1 trailer does not match the pickle body (truncated or corrupted file)")
        raw = body
    return _NumpyOnlyUnpickler(io.BytesIO(raw)).load()


def write_reference_ckpt(ckpt, path):
    body = pickle.dumps(_to_numpy(ckpt), 4)
    with open(path, "wb") as f:
        f.write(body + hashlib.sha1(body).digest() + _TAG)


def _to_numpy(x):
    if isinstance(x, dict):
        return {k: _to_numpy(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_to_numpy(v) for v in x)
    if hasattr(x, "detach") and hasattr(x, "cpu"):                       # torch tensor (kept optional: no torch import here)
        return x.detach().cpu().numpy()
    return x


# ---------------------------------------------------------------------------------------------------- parameters
def _linear_to_flat(ws):
    """[W (out,in) ...] of an nn.Sequential(Linear, ReLU, ...) -> flat (out,in)-row-major vector with the last layer padded
    to 16 rows -- FullyFusedMlp_weight.__init__ stores weights (in,out), pads columns to 16 and flattens the transpose
    (fully_fused_mlp.py:26-40); nn.Linear already keeps (out,in)."""
    ws = [np.asarray(w) for w in ws]
    last = ws[-1]
    if last.shape[0] < 16:
        last = np.concatenate([last, np.zeros((16 - last.shape[0], last.shape[1]), last.dtype)], 0)
    return np.concatenate([w.reshape(-1) for w in ws[:-1]] + [last.reshape(-1)])


def _flat_to_linear(flat, n_hidden_matmuls, n_out):
    shapes = [(64, 32)] + [(64, 64)] * n_hidden_matmuls + [(16, 64)]
    out, o = [], 0
    for s in shapes:
        out.append(np.asarray(flat[o:o + s[0] * s[1]]).reshape(s))
        o += s[0] * s[1]
    out[-1] = out[-1][:n_out]
    return out


def model_params_from_reference(model_sd, n_table):
    """-> {'m_grid', 'density', 'rgb'} numpy arrays (dtype as stored) from the reference's model.state_dict()."""
    by_size = {}
    for k, v in model_sd.items():
        v = np.asarray(v)
        by_size.setdefault(v.size, []).append((k, v))
    out = {}
    grid = [kv for kv in by_size.get(n_table, []) if "grid" in kv[0]] or by_size.get(n_table, [])
    if not grid:
        raise KeyError(f"no tensor with {n_table} elements (the hash table for this aabb_scale) in the checkpoint's model dict: "
                       f"{sorted((k, np.asarray(v).shape) for k, v in model_sd.items())[:12]}")
    out["m_grid"] = grid[0][1].reshape(-1)
    for name, n, nhm, n_out in (("density", N_DENSITY, 0, 16), ("rgb", N_RGB, 1, 3)):
        hit = [kv for kv in by_size.get(n, []) if "con_weights" in kv[0]]
        if hit:
            out[name] = hit[0][1].reshape(-1)
            continue
        prefix = "density_mlp." if name == "density" else "rgb_mlp."
        lin = sorted((k, np.asarray(v)) for k, v in model_sd.items() if k.startswith(prefix) and k.endswith(".weight"))
        if len(lin) != nhm + 2:
            raise KeyError(f"neither {prefix}con_weights ({n} elements) nor {nhm + 2} {prefix}<i>.weight matrices in the checkpoint")
        out[name] = _linear_to_flat([w for _, w in lin])
    return out


def _by_size(tensors, sizes):
    """Pick, for every wanted size, the tensor of a list with that element count."""
    got = {}
    for t in tensors:
        t = np.asarray(t)
        if t.size in sizes and t.size not in got:
            got[t.size] = t.reshape(-1)
    missing = [s for s in sizes if s not in got]
    if missing:
        raise KeyError(f"optimizer state without tensors of {missing} elements")
    return [got[s] for s in sizes]


def _floor_second_moments(m, v):
    """A reference-written file holds moments in the parameter dtype: with fp16, second moments below fp16's smallest subnormal
    (6e-8) are stored as 0 while the first moment survives, and lr * m / (sqrt(0) + 1e-15) would throw the entry to inf on the next
    step.  Floor v at m^2 (|update| <= lr, Adam's own bound) for exactly those entries; where m^2 underflows fp32 as well, drop the
    momentum.  -> (m, v) lists in fp32."""
    fixed = []
    for mm, vv in zip(m, v):
        mm32, vv32 = np.asarray(mm, np.float32), np.asarray(vv, np.float32).copy()
        bad = (vv32 == 0) & (mm32 != 0)
        vv32[bad] = mm32[bad] * mm32[bad]
        still = bad & (vv32 == 0)
        if still.any():
            mm32 = mm32.copy()
            mm32[still] = 0
        fixed.append((mm32, vv32))
    return [f[0] for f in fixed], [f[1] for f in fixed]


# ---------------------------------------------------------------------------------------------------- whole checkpoints
def reference_to_native(ref, n_table):
    """Reference params.pkl dict -> the dict Runner.load_ckpt consumes (numpy arrays; the loader moves them to the device).
    Parameter order: [m_grid, density_mlp.con_weights, rgb_mlp.con_weights] (NGPNetworks.parameters())."""
    p = model_params_from_reference(ref["model"], n_table)
    sizes = [n_table, N_DENSITY, N_RGB]
    nested = ref["nested_optimizer"]["defaults"]
    pg = nested["param_groups"][0]
    ema_d = ref["ema_optimizer"]["defaults"]
    try:
        if "values_f32" in pg:
            # written by native_to_reference: the fp32 optimizer state next to the parameter-dtype copies the reference reads
            v = _by_size(pg["values_f32"], sizes)
            m = _by_size(pg["m_f32"], sizes)
            ema_vals = _by_size(ema_d["param_groups"][0].get("values_f32", ema_d["param_groups"][0]["values"]), sizes)
        else:
            v = _by_size(pg["values"], sizes)
            m = _by_size(pg["m"], sizes)
            ema_vals = _by_size(ema_d["param_groups"][0]["values"], sizes)
            m, v = _floor_second_moments(m, v)
    except KeyError:
        # nn.Linear checkpoints keep one moment tensor per matrix; the flat fused layout restarts the moments and takes the
        # parameters themselves as EMA values (after every ema_step the two are equal, ema.py:33-36)
        m = [np.zeros(n, np.float32) for n in sizes]
        v = [np.zeros(n, np.float32) for n in sizes]
        ema_vals = [p["m_grid"], p["density"], p["rgb"]]
    model = {"pos_encoder.m_grid": p["m_grid"], "density_mlp.con_weights": p["density"], "rgb_mlp.con_weights": p["rgb"]}
    return _native_dict(ref, model, m, v, ema_vals)


def _native_dict(ref, model, m, v, master):
    """The native checkpoint dict around the model dict and the optimizer lists (in the model's parameter order)."""
    nested = ref["nested_optimizer"]["defaults"]
    ema_d = ref["ema_optimizer"]["defaults"]
    steps = int(ema_d["steps"])
    opt = ref["optimizer"]["defaults"]
    s = ref["sampler"]
    mean = np.asarray(s["density_grid_mean"], np.float32).reshape(-1)[:1]
    sampler = {"density_grid": np.asarray(s["density_grid"], np.float32).reshape(-1),
               "density_grid_bitfield": np.asarray(s["density_grid_bitfield"], np.uint8).reshape(-1),
               "density_grid_mean": mean, "density_grid_ema_step": np.asarray(s["density_grid_ema_step"], np.int32).reshape(-1)[:1]}
    if "n_rays_per_batch" in s:
        sampler["n_rays_per_batch"] = int(np.asarray(s["n_rays_per_batch"]).reshape(-1)[0])
    if "rng" in s:
        sampler["rng"] = np.asarray(s["rng"], np.int64).reshape(-1)
    f32 = lambda a: np.asarray(a, np.float32)                                            # noqa: E731
    return {
        "global_step": int(ref["global_step"]),
        "model": model,
        "sampler": sampler,
        "optimizer": {"steps": int(opt["steps"]), "m_learning_rate_factor": float(opt["m_learning_rate_factor"])},
        "nested_optimizer": {"n_step": steps, "lr": float(nested.get("lr", 0.1)), "m": [f32(x) for x in m], "v": [f32(x) for x in v],
                             "master": [f32(x) for x in master]},
        "ema_optimizer": {"steps": steps, "decay": float(ema_d.get("decay", 0.95))},
    }


def native_to_reference(nat, adam_hyper=None, expdecay_hyper=None, param_dtype=np.float16):
    """The dict Runner.save_ckpt builds (tensors or arrays) -> the reference's params.pkl structure (numpy)."""
    nat = _to_numpy(nat)
    model = {k: np.asarray(v) for k, v in nat["model"].items()}
    order = ["pos_encoder.m_grid", "density_mlp.con_weights", "rgb_mlp.con_weights"]
    nested = nat["nested_optimizer"]
    return _reference_dict(nat, {k: model[k] for k in order}, nested["m"], nested["v"], nested["master"], adam_hyper, expdecay_hyper, param_dtype)


def _reference_dict(nat, model, m, v, master, adam_hyper, expdecay_hyper, param_dtype):
    """The reference's params.pkl structure around its model dict and the optimizer lists (one entry per model key, in its order);
    nat: the native dict (numpy) the counters, learning rates and sampler state come from."""
    nested, ema = nat["nested_optimizer"], nat["ema_optimizer"]
    cast = lambda a: np.asarray(a).astype(param_dtype)                                   # noqa: E731  Jittor keeps m / values in the parameter dtype
    f32 = lambda a: np.asarray(a, np.float32)                                            # noqa: E731
    hyper = dict(lr=float(nested["lr"]), eps=1e-15, betas=(0.9, 0.99), weight_decay=0)
    hyper.update(adam_hyper or {})
    dec = dict(base_lr=hyper["lr"], decay_start=20000, decay_interval=10000, decay_base=0.33, decay_end=10000000)
    dec.update(expdecay_hyper or {})
    s = nat["sampler"]
    mean = np.zeros(16384, np.float32)                                                   # density_grid_sampler.py:91-92: div_round_up(128^3, 128) slots
    mean[0] = float(np.asarray(s["density_grid_mean"]).reshape(-1)[0])
    sampler = {"density_grid": np.asarray(s["density_grid"], np.float32), "density_grid_bitfield": np.asarray(s["density_grid_bitfield"], np.uint8),
               "density_grid_mean": mean, "density_grid_ema_step": np.asarray(s["density_grid_ema_step"], np.int32).reshape(1)}
    for k in ("n_rays_per_batch", "rng"):
        if k in s:
            sampler[k] = np.asarray(s[k])
    return {
        "global_step": int(nat["global_step"]),
        "model": model,
        "sampler": sampler,
        "optimizer": {"defaults": dict(dec, steps=int(nat["optimizer"]["steps"]), m_learning_rate_factor=nat["optimizer"]["m_learning_rate_factor"])},
        # "values"/"m" in the parameter dtype are what the reference's load_ckpt reads (runner.py:133-151); the *_f32 keys are ignored
        # by it and preferred by reference_to_native, so a save -> load in this repo is lossless (fp16 flushes most second moments to 0)
        "nested_optimizer": {"defaults": dict(hyper, param_groups=[{"values": [cast(x) for x in v], "m": [cast(x) for x in m],
                                                                    "values_f32": [f32(x) for x in v], "m_f32": [f32(x) for x in m]}])},
        "ema_optimizer": {"defaults": {"lr": 0, "decay": float(ema["decay"]), "steps": int(ema["steps"]),
                                       "param_groups": [{"values": [cast(x) for x in master],
                                                         "values_f32": [f32(x) for x in master]}]}},
    }


# ---------------------------------------------------------------------------------------------------- vanilla NeRF (OriginNeRFNetworks)
def nerf_reference_shapes():
    """{reference key: shape} of OriginNeRFNetworks' 24 tensors in its state_dict() order (ori_nerf_network.py:21-26)."""
    from ..plugin.nerf import REF_LAYERS, REF_ORDER
    return {f"{name}.{part}": (REF_LAYERS[name][0] if part == "weight" else REF_LAYERS[name][0][:1]) for name in REF_ORDER for part in ("weight", "bias")}


def _nerf_split(entries, flat):
    """Native NeRF tensors -> {reference key: fp32 array of the reference shape}.  flat: entries is [the one flat vector of the fp16
    kernels' layout] (mapped through plugin/nerf.py's unpack); else one entry per reference key, in nerf_reference_shapes() order."""
    shapes = nerf_reference_shapes()
    if not flat:
        return {k: np.asarray(e, np.float32).reshape(shp) for (k, shp), e in zip(shapes.items(), entries)}
    import torch
    from ..plugin.nerf import unpack
    out = {}
    for name, (W, b) in unpack(torch.from_numpy(np.ascontiguousarray(np.asarray(entries[0])).reshape(-1))).items():
        out[f"{name}.weight"], out[f"{name}.bias"] = W.numpy(), b.numpy()
    return {k: out[k] for k in shapes}


def _nerf_join(tensors, flat, half=False):
    """Inverse of _nerf_split: {reference key: array} -> [one flat vector, fp16 if half else fp32, zero padding] (flat) or one flat fp32
    entry per key."""
    if not flat:
        return [np.asarray(t, np.float32).reshape(-1) for t in tensors.values()]
    import torch
    from ..plugin.nerf import REF_ORDER, pack
    t = {name: (torch.from_numpy(np.asarray(tensors[f"{name}.weight"], np.float32)), torch.from_numpy(np.asarray(tensors[f"{name}.bias"], np.float32)))
         for name in REF_ORDER}
    return [pack(t, dtype=torch.float16 if half else torch.float32).numpy()]


def nerf_native_to_reference(nat, adam_hyper=None, expdecay_hyper=None, param_dtype=np.float16):
    """native_to_reference for OriginNeRFNetworks: the model dict and every optimizer list as the reference's 24 tensors by name, from
    either native form (fp16: the flat `params` vector and flat moments; fp32: the nn.Linear chain, already under the reference names)."""
    nat = _to_numpy(nat)
    flat = "params" in nat["model"]
    model = _nerf_split(list(nat["model"].values()), flat)
    nested = nat["nested_optimizer"]
    m, v, master = (list(_nerf_split(nested[k], flat).values()) for k in ("m", "v", "master"))
    return _reference_dict(nat, {k: t.astype(param_dtype) for k, t in model.items()}, m, v, master, adam_hyper, expdecay_hyper, param_dtype)


def nerf_reference_to_native(ref, fp16):
    """A params.pkl of OriginNeRFNetworks -> the native dict of the fp16 kernels' model (fp16=True: the flat `params` vector and flat
    fp32 moments, zero padding) or of the nn.Linear chain (fp16=False).  Tensors are matched by name: the i-th entry of the Adam and
    EMA lists belongs to the i-th key of the model dict, and each must have that key's shape."""
    model = ref["model"]
    keys = list(model)
    shapes = nerf_reference_shapes()
    missing = [k for k in shapes if k not in model]
    if missing:
        raise KeyError(f"the checkpoint's model dict is not OriginNeRFNetworks' (D=8, W=256, skips=[4]): no {missing[:3]}"
                       f"{' ...' if len(missing) > 3 else ''}; it holds {keys[:4]}{' ...' if len(keys) > 4 else ''}")
    for k, shp in shapes.items():
        if tuple(np.shape(model[k])) != shp:
            raise ValueError(f"params.pkl: model tensor {k} has shape {tuple(np.shape(model[k]))}, OriginNeRFNetworks' is {shp}")
    pg = ref["nested_optimizer"]["defaults"]["param_groups"][0]
    ema_pg = ref["ema_optimizer"]["defaults"]["param_groups"][0]
    lossless = "values_f32" in pg                                      # written by nerf_native_to_reference

    def by_key(what, lst):
        if len(lst) != len(keys):
            raise ValueError(f"params.pkl: {what} holds {len(lst)} tensors, the model dict {len(keys)}")
        for k, t in zip(keys, lst):
            if tuple(np.shape(t)) != tuple(np.shape(model[k])):
                raise ValueError(f"params.pkl: the {what} entry of {k} has shape {tuple(np.shape(t))}, the parameter {tuple(np.shape(model[k]))}")
        got = dict(zip(keys, lst))
        return [np.asarray(got[k], np.float32) for k in shapes]

    if lossless:
        v, m = by_key("Adam values_f32", pg["values_f32"]), by_key("Adam m_f32", pg["m_f32"])
        master = by_key("EMA values_f32", ema_pg.get("values_f32", ema_pg["values"]))
    else:
        m, v = _floor_second_moments(by_key("Adam m", pg["m"]), by_key("Adam values", pg["values"]))
        master = by_key("EMA values", ema_pg["values"])
    params = {k: np.asarray(model[k]) for k in shapes}
    if fp16:
        native_model = {"params": _nerf_join(params, True, half=True)[0]}
    else:
        native_model = {k: t.astype(np.float32) for k, t in params.items()}
    lists = [_nerf_join(dict(zip(shapes, x)), fp16) for x in (m, v, master)]
    return _native_dict(ref, native_model, *lists)


def load_native_from_reference_file(path, n_table, device, model_dtypes=None, nerf_fp16=None):
    """params.pkl -> the dict Runner.load_ckpt consumes, with torch tensors on `device` (model tensors cast to model_dtypes[key]).
    nerf_fp16: None for NGPNetworks (hash table of n_table entries); True / False for OriginNeRFNetworks with that fp16 setting."""
    import torch
    ref = read_reference_ckpt(path)
    nat = reference_to_native(ref, n_table) if nerf_fp16 is None else nerf_reference_to_native(ref, nerf_fp16)

    def dev(x):
        if isinstance(x, np.ndarray):
            return torch.from_numpy(np.ascontiguousarray(x)).to(device)
        if isinstance(x, list):
            return [dev(t) for t in x]
        if isinstance(x, dict):
            return {k: dev(v) for k, v in x.items()}
        return x

    ck = dev(nat)
    if model_dtypes:
        ck["model"] = {k: v.to(model_dtypes[k]) for k, v in ck["model"].items()}
    return ck
