"""The `jt.code` glue a JNeRF checkout needs to run `projects/ngp` on libngp_b200.so: drop-in replacements for the bodies of the
reference's operator classes, same class names, constructor arguments and execute / grad signatures, each `cuda_src` a one-line call
of the C ABI (include/ngp_b200.h).  INTEGRATION.md explains the mapping operator by operator.

Jittor is imported lazily: the module always imports (tests type-check every CUDA snippet below against the header with the host
compiler, tests/test_integration_stubs.py), the classes need `import jittor` at construction time.  Usage inside JNeRF:

    from jnerf_b200 import jittor_glue as glue
    glue.configure("/path/to/repo")                      # where include/ and jnerf_b200/libngp_b200.so live
    # models/position_encoders/hash_encoder/grid_encode.py:     GridEncode = glue.GridEncode
    # models/position_encoders/sh_encoder/sh_encoder.py:        body of SHEncoder.execute = glue.sh_encode
    # ops/code_ops/fully_fused_mlp.py:                          FullyFusedMlp_weight = glue.FullyFusedMlp_weight
    # models/samplers/density_grid_sampler/ray_sampler.py ...:  glue.ray_march / glue.compact / glue.CalcRgb
"""
import os

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NGP_LIB = os.path.join(_ROOT, "jnerf_b200", "libngp_b200.so")
NGP_INC = os.path.join(_ROOT, "include")

CUDA_HEADER = ('#include "ngp_b200.h"\n#include <stdexcept>\n'
               '#define NGP_OK(x) do { if ((x) != 0) throw std::runtime_error(ngp_last_error()); } while (0)\n')

# ---- the CUDA bodies (host C++ launched on stream 0, as every jt.code op of the reference; inK_p / outK_p / inK_shapeJ are the
# names jt.code injects) -----------------------------------------------------------------------------------------------------
SRC = {
    # models/position_encoders/hash_encoder/grid_encode.py:66-190
    "hash_fwd": "NGP_OK(ngp_hash_fwd(0, in0_shape0, in0_p, in1_p, sizeof(in1_type) == 2 ? NGP_F16 : NGP_F32, in2_p, out_p));",
    "hash_bwd": "NGP_OK(ngp_hash_bwd(0, in0_shape0, in0_p, in1_p, sizeof(in1_type) == 2 ? NGP_F16 : NGP_F32, in2_p, out_p, out->num));",
    # models/position_encoders/sh_encoder/sh_encoder.py:26-53
    "sh_fwd": "NGP_OK(ngp_sh_fwd(0, in0_shape0, in0_p, sizeof(out_type) == 2 ? NGP_F16 : NGP_F32, out_p));",
    # ops/code_ops/fully_fused_mlp.py:42-145 ({nhm} = hidden matmuls = len(weights) - 2, {nout} = output_shape1)
    "mlp_fwd": "NGP_OK(ngp_mlp_fwd(0, in1_p, in0_p, out1_p, out0_p, {nhm}, in0_shape0));",
    "mlp_bwd": "NGP_OK(ngp_mlp_bwd(0, in0_p, in1_p, in2_p, in3_p, out0_p, nullptr, out1_p, {nhm}, {nout}, in1_shape0));",
    # models/networks/ngp_network.py:77-89 as one fused op over the sampler's (N,7) coordinate rows
    "network_fwd": "NGP_OK(ngp_network_fwd(0, in0_shape0, nullptr, in0_p, in1_p, in2_p, in3_p, in4_p, out0_p, out1_p));",
    "network_bwd": "NGP_OK(ngp_network_bwd(0, in0_shape0, nullptr, in0_p, in1_p, in2_p, in3_p, in4_p, in5_p, out0_p, out1_p, out2_p));",
    "density_fwd": "NGP_OK(ngp_density_fwd(0, in0_shape0, in0_p, in1_p, in2_p, in3_p, out_p));",
    # models/samplers/density_grid_sampler/ray_sampler.py:20-72, compacted_coord.py:28-70
    "march": ("NGP_OK(ngp_march(0, in0_shape0, {aabb0}, {aabb1}, out0_shape0, in0_p, in1_p, (const uint8_t*)in2_p, {cone}, {near}, NERF_CASCADES(), "
              "{const_dt}, rng.state, rng.inc, (uint32_t*)out3_p, (uint32_t*)out1_p, (uint32_t*)out2_p, out0_p, in3_p)); rng.advance();"),
    "compact": "NGP_OK(ngp_compact(0, in1_shape0, out0_shape0, in0_p, (uint32_t*)in1_p, out0_p, (uint32_t*)out1_p, (uint32_t*)out2_p, 1));",
    # models/samplers/density_grid_sampler/calc_rgb.py:31-147
    "composite_fwd": "NGP_OK(ngp_composite_fwd(0, in2_shape0, in0_p, {dtype}, in1_p, (uint32_t*)in2_p, (uint32_t*)in3_p, in4_p, NERF_CASCADES(), out0_p));",
    "composite_bwd": ("NGP_OK(ngp_composite_bwd(0, in2_shape0, in0_shape0, in0_p, {dtype}, in1_p, (uint32_t*)in2_p, in3_p, in4_p, in5_p, NERF_CASCADES(), "
                      "out0_p));"),
    "composite_infer": "NGP_OK(ngp_composite_infer(0, in2_shape0, in0_p, {dtype}, in1_p, (uint32_t*)in2_p, NERF_CASCADES(), out0_p, out1_p));",
    # mark_untrained_density_grid.py, generate_grid_samples_nerf_nonuniform.py, splat_grid_samples_nerf_max_nearest_neighbor.py,
    # ema_grid_samples_nerf.py, update_bitfield.py
    "grid_mark_untrained": "NGP_OK(ngp_grid_mark_untrained(0, out0_shape0, out0_p, in0_shape0, in0_p, in1_p, {W}, {H}));",
    "grid_generate_samples": ("NGP_OK(ngp_grid_generate_samples(0, out1_shape0, rng.state, rng.inc, (uint32_t*)in1_p, {aabb0}, {aabb1}, in0_p, out0_p, "
                              "(uint32_t*)out1_p, {n_cascades}, {thresh})); rng.advance();"),
    "grid_splat": "NGP_OK(ngp_grid_splat(0, in0_shape0, (uint32_t*)in0_p, in1_p, {dtype}, out0_p));",
    "grid_ema": "NGP_OK(ngp_grid_ema(0, out0_shape0, (float){decay}, out0_p, in0_p));",
    "grid_update_bitfield": "NGP_OK(ngp_grid_update_bitfield(0, in0_p, out1_p, (uint8_t*)out0_p, NERF_CASCADES()));",
    # optims/adam.py + optims/ema.py in one sweep per parameter tensor
    "adam_ema": "NGP_OK(ngp_adam_ema(0, in0_shape0, in0_p, NGP_F16, in1_p, NGP_F16, 1.0f, in2_p, in3_p, in4_p, (float){lr}, 0.9f, 0.99f, 1e-15f, {step}, 0.95f, 1));",
    # contrib/plenoxel: volume_render_cuvol.py (forward, and forward + MSE + backward fused), tv_grad_sparse.py, optims/svox2_optim.py,
    # sample_grid.py, grid_weight_render.py, dilate.py and the link rebuild of svox2_network.py:470-482 (xform_p: offset[3] + scaling[3],
    # opts_p: step, sigma_thresh, stop_thresh, background, host float arrays declared before the call)
    "svox_train_step": ("NGP_OK(ngp_svox_train_step(0, in0_shape0, in0_p, {W}, {H}, in1_p, {fx}, {fy}, {cx}, {cy}, (const uint8_t*)in2_p, in3_p, "
                        "in3_shape0, in3_shape1, in3_shape2, in4_p, in5_p, xform_p, opts_p, out0_p, out1_p, out2_p, out3_p));"),
    "svox_render": ("NGP_OK(ngp_svox_render(0, out0_shape0, {first}, {W}, in0_p, {fx}, {fy}, {cx}, {cy}, in1_p, in1_shape0, in1_shape1, in1_shape2, "
                    "in2_p, in3_p, xform_p, opts_p, out0_p));"),
    "svox_tv_grad": ("NGP_OK(ngp_svox_tv_grad(0, in0_p, in0_shape0, in0_shape1, in0_shape2, in1_p, in1_shape1, {start}, {n_cells}, (float){scale}, "
                     "{ignore_edge}, out0_p, out1_p));"),
    "svox_rmsprop": ("NGP_OK(ngp_svox_rmsprop(0, in0_shape0, in1_shape0 * in1_shape1, in0_p, in1_p, in2_p, in3_p, in4_p, in5_p, (float){lr_sigma}, "
                     "(float){lr_sh}, 0.95f, 0.95f, 1e-8f));"),
    "svox_sample": ("NGP_OK(ngp_svox_sample(0, in0_shape0, in0_p, in1_p, in1_shape0, in1_shape1, in1_shape2, in2_p, in3_p, {want_sh}, out0_p, "
                    "out1_p));"),
    "svox_weight_render": ("NGP_OK(ngp_svox_weight_render(0, {W}, {H}, in1_p, {fx}, {fy}, {cx}, {cy}, in0_p, in0_shape0, in0_shape1, in0_shape2, "
                           "xform_p, 0.5f, 0.2f, out0_p));"),
    "svox_dilate": "NGP_OK(ngp_svox_dilate(0, in0_shape0, in0_shape1, in0_shape2, (const uint8_t*)in0_p, (uint8_t*)out0_p));",
    "svox_compact": ("NGP_OK(ngp_svox_compact(0, in0_shape0, in0_shape1, in0_shape2, (const uint8_t*)in0_p, in1_p, lattice_p, out1_shape0, out3_p, "
                     "out0_p, out1_p, out2_p));"),
}


def configure(repo_root):
    """Point the glue at a checkout / install of this repository."""
    global NGP_LIB, NGP_INC
    NGP_LIB = os.path.join(repo_root, "jnerf_b200", "libngp_b200.so")
    NGP_INC = os.path.join(repo_root, "include")


def ngp_options():
    """compile_options that make a jt.code module find the header and link the library, the way the reference links its prebuilt MLP
    object (ops/code_ops/fully_fused_mlp.py:84)."""
    return {f"FLAGS: -I{NGP_INC} -Xlinker {NGP_LIB} -Xlinker -rpath -Xlinker {os.path.dirname(NGP_LIB)} ": 1}


def _jt():
    try:
        import jittor as jt
    except ImportError as e:                                         # pragma: no cover - Jittor is not part of this image
        raise ImportError("jnerf_b200.jittor_glue builds jt.code operators and needs Jittor; "
                          "without it use the torch-hosted mirror jnerf_b200.plugin") from e
    return jt


def _code(shapes, dtypes, inputs, src, header=CUDA_HEADER):
    jt = _jt()
    out = jt.code(shapes, dtypes, inputs, cuda_header=header, cuda_src=src)
    for o in (out if isinstance(out, (list, tuple)) else [out]):
        o.compile_options = ngp_options()
    return out


def level_table(aabb_scale=1, n_levels=16, base_resolution=16, log2_hashmap_size=19, primes=(1, 19349663, 83492791)):
    """One-time 512-byte level table (replaces m_hashmap_offsets_table and the exp2f of every kernel): filled by the two host entry
    points through ctypes, uploaded as a uint8 Var."""
    import ctypes as C
    import numpy as np
    jt = _jt()
    lib = C.CDLL(NGP_LIB)
    offsets = np.zeros(n_levels + 1, np.uint32)
    pls = C.c_double()
    lib.ngp_hash_offsets.argtypes = [C.c_double, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    assert lib.ngp_hash_offsets(float(aabb_scale), n_levels, base_resolution, log2_hashmap_size, offsets.ctypes.data, C.addressof(pls)) == 0
    table = jt.zeros([n_levels * 32], "uint8")
    jt.sync_all()
    lib.ngp_hash_level_table_primes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32, C.c_float, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    assert lib.ngp_hash_level_table_primes(None, offsets.ctypes.data, n_levels, base_resolution, float(np.float32(np.log2(pls.value))),
                                           C.c_void_p(table.data_ptr() if hasattr(table, "data_ptr") else 0), *[int(p) for p in primes]) == 0
    return table, int(offsets[-1]) * 2


class GridEncode:
    """models/position_encoders/hash_encoder/grid_encode.py:11-190 (a jt.Function in the reference)."""

    def __new__(cls, *a, **k):
        jt = _jt()

        class _GridEncode(jt.Function):
            def __init__(self, hash_func_header, aabb_scale=1, n_pos_dims=3, n_features_per_level=2, n_levels=16, base_resolution=16,
                         log2_hashmap_size=19, n_rays_per_batch=4096, MAX_STEP=1024, using_fp16=False):
                from .plugin.encoders import DEFAULT_HASH, parse_hash_func
                expr = hash_func_header.split(")", 1)[1] if "get_index" in hash_func_header else hash_func_header
                self.levels, self.m_n_params = level_table(aabb_scale, n_levels, base_resolution, log2_hashmap_size,
                                                           parse_hash_func(expr.strip() or DEFAULT_HASH))
                self.grad_type = "float16" if using_fp16 else "float32"

            def execute(self, x, m_grid):
                self.x = x
                return _code([x.shape[0], 32], m_grid.dtype, [x, m_grid, self.levels], SRC["hash_fwd"])

            def grad(self, grad_x):
                return None, _code([self.m_n_params], grad_x.dtype, [self.x, grad_x, self.levels], SRC["hash_bwd"])
        return _GridEncode(*a, **k)


def sh_encode(x, grad_type="float16"):
    """models/position_encoders/sh_encoder/sh_encoder.py:26-53."""
    _jt()
    return _code((x.shape[0], 16), grad_type, [x], SRC["sh_fwd"])


class FullyFusedMlp_weight:
    """ops/code_ops/fully_fused_mlp.py:42-145: con_weights is the flat fp16 parameter vector of FMLP."""

    def __new__(cls, *a, **k):
        jt = _jt()

        class _FFMLP(jt.Function):
            def __init__(self, weights, check_mid="0", output_activation="None"):
                self.nhm = len(weights) - 2
                self.width = weights[0].shape[0]
                self.output_shape1 = weights[-1].shape[0]
                self.n_params = sum(w.numel() for w in weights[:-1]) + 16 * self.width

            def execute(self, a, con_weights):
                B = a.shape[0]
                self.input, self.con_weights = a, con_weights
                self.outputs, self.output_intermediate = _code([(B, 16), (B * (self.nhm + 1), self.width)], [a.dtype, a.dtype], [a, con_weights],
                                                               SRC["mlp_fwd"].format(nhm=self.nhm))
                return self.outputs[:, :self.output_shape1]

            def grad(self, grads):
                jt_ = _jt()
                B = grads.shape[0]
                dy = jt_.concat([grads, jt_.zeros((B, 16 - grads.shape[1]), grads.dtype)], 1) if grads.shape[1] < 16 else grads
                dX, dW = _code([(B, 32), (self.n_params,)], [grads.dtype, "float32"], [self.con_weights, self.input, self.output_intermediate, dy],
                               SRC["mlp_bwd"].format(nhm=self.nhm, nout=self.output_shape1))
                return dX, dW.cast(self.con_weights.dtype)
        return _FFMLP(*a, **k)


def network_fwd(coords, m_grid, levels, wd, wr):
    """models/networks/ngp_network.py:77-84 fused: (N,7) NerfCoordinate rows -> ((N,4) fp16 {r,g,b,sigma_raw}, (N,32) encoded features)."""
    _jt()
    N = coords.shape[0]
    return _code([(N, 4), (N, 32)], ["float16", "float16"], [coords, m_grid, levels, wd, wr], SRC["network_fwd"])


def network_bwd(coords, enc, levels, wd, wr, dout, n_grid_params):
    """Backward of network_fwd: gradients of the hash table (fp16) and of both weight vectors (fp32); outputs are zero-initialised."""
    jt = _jt()
    outs = [jt.zeros([n_grid_params], "float16"), jt.zeros([wd.numel()], "float32"), jt.zeros([wr.numel()], "float32")]
    return jt.code(inputs=[coords, enc, levels, wd, wr, dout], outputs=outs, cuda_header=CUDA_HEADER, cuda_src=SRC["network_bwd"])


def ray_march(rays_o, rays_d, bitfield, workspace, coords_out, rays_index, rays_numsteps, counter, aabb_range, cone_angle_constant, near_distance,
              const_dt, global_headers=""):
    """RaySampler.execute (ray_sampler.py:20-72): no 117 MB memset, no .item(); `global_headers` = the reference's proj_options header
    that declares jittor::rng and NERF_CASCADES()."""
    jt = _jt()
    src = SRC["march"].format(aabb0=float(aabb_range[0]), aabb1=float(aabb_range[1]), cone=float(cone_angle_constant), near=float(near_distance),
                              const_dt=int(bool(const_dt)))
    return jt.code(inputs=[rays_o, rays_d, bitfield, workspace], outputs=[coords_out, rays_index, rays_numsteps, counter],
                   cuda_header=global_headers + CUDA_HEADER, cuda_src=src)


def compact(coords_in, numsteps_in, coords_out, numsteps_out, counters):
    """CompactedCoord.execute (compacted_coord.py:28-70); pass coords_in as coords_out to make it bookkeeping-only."""
    jt = _jt()
    return jt.code(inputs=[coords_in, numsteps_in], outputs=[coords_out, numsteps_out, counters], cuda_header=CUDA_HEADER, cuda_src=SRC["compact"])


class CalcRgb:
    """models/samplers/density_grid_sampler/calc_rgb.py:31-147."""

    def __new__(cls, *a, **k):
        jt = _jt()

        class _CalcRgb(jt.Function):
            def __init__(self, density_grid_mean, global_headers=""):
                self.density_grid_mean, self.header = density_grid_mean, global_headers + CUDA_HEADER

            def execute(self, network_output, coords_in, rays_numsteps, rays_numsteps_compacted, training_background_color):
                self.saved = (network_output, coords_in, rays_numsteps_compacted)
                dtype = "NGP_F16" if str(network_output.dtype) == "float16" else "NGP_F32"
                self.rgb = jt.code([rays_numsteps.shape[0], 3], "float32", [network_output, coords_in, rays_numsteps, rays_numsteps_compacted,
                                                                           training_background_color],
                                   cuda_header=self.header, cuda_src=SRC["composite_fwd"].format(dtype=dtype))
                return self.rgb

            def grad(self, grad_x):
                net, coords, ns_c = self.saved
                dtype = "NGP_F16" if str(net.dtype) == "float16" else "NGP_F32"
                dnet = jt.code(net.shape, net.dtype, [net, coords, ns_c, grad_x, self.rgb, self.density_grid_mean], cuda_header=self.header,
                               cuda_src=SRC["composite_bwd"].format(dtype=dtype))
                return dnet, None, None, None, None

            def inference(self, network_output, coords_in, rays_numsteps):
                dtype = "NGP_F16" if str(network_output.dtype) == "float16" else "NGP_F32"
                R = rays_numsteps.shape[0]
                return jt.code([(R, 3), (R, 1)], ["float32", "float32"], [network_output, coords_in, rays_numsteps], cuda_header=self.header,
                               cuda_src=SRC["composite_infer"].format(dtype=dtype))
        return _CalcRgb(*a, **k)


def adam_ema(param, grad, m, v, master, lr, step):
    """optims/adam.py + optims/ema.py in one sweep (in place on all five tensors)."""
    jt = _jt()
    return jt.code(inputs=[param, grad, m, v, master], outputs=[param], cuda_header=CUDA_HEADER, cuda_src=SRC["adam_ema"].format(lr=float(lr), step=int(step)))
