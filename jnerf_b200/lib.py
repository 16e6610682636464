"""ctypes binding of libngp_b200.so (include/ngp_b200.h).  Fails loudly when the CUDA library is missing or a call
returns an error -- there is no CPU fallback anywhere in the product path."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NGP_B200_LIB") or os.path.join(HERE, "libngp_b200.so")   # override: A/B timing of experimental builds

_vp, _u32, _u64, _i64, _f32, _i32, _f64 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int64, C.c_float, C.c_int, C.c_double

# name -> (restype, argtypes); mirrors include/ngp_b200.h one to one
SIGNATURES = {
    "ngp_last_error": (C.c_char_p, []),
    "ngp_version": (_i32, []),
    "ngp_sm_count": (_i32, []),
    "ngp_debug_timeout_flag": (_i32, []),
    "ngp_hash_offsets": (_i32, [_f64, _i32, _i32, _i32, _vp, _vp]),
    "ngp_hash_level_table": (_i32, [_vp, _vp, _i32, _u32, _f32, _vp]),
    "ngp_hash_level_table_primes": (_i32, [_vp, _vp, _i32, _u32, _f32, _vp, _u32, _u32, _u32]),
    "ngp_hash_fwd": (_i32, [_vp, _u32, _vp, _vp, _i32, _vp, _vp]),
    "ngp_hash_bwd": (_i32, [_vp, _u32, _vp, _vp, _i32, _vp, _vp, _u64]),
    "ngp_sh_fwd": (_i32, [_vp, _u32, _vp, _i32, _vp]),
    "ngp_mlp_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "ngp_mlp_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32]),
    "ngp_mlp_bwd_dgrad": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32]),
    "ngp_mlp_param_count": (_i32, [_u32]),
    "ngp_network_fwd": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_network_bwd": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_network_bwd_fx_bytes": (_i32, [_u64, _vp, _vp]),
    "ngp_network_bwd_fx": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _u64, _vp, _u64]),
    "ngp_density_fwd": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    "ngp_nerf_param_count": (_i32, [_vp]),
    "ngp_nerf_workspace_bytes": (_i32, [_u32, _vp, _vp]),
    "ngp_nerf_fwd": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    "ngp_nerf_density": (_i32, [_vp, _u32, _vp, _vp, _vp]),
    "ngp_nerf_bwd": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_mip_rays": (_i32, [_vp, _u32, _vp, _u32, _u32, _vp, _f32, _f32, _f32, _vp, _vp, _vp]),
    "ngp_mip_sample": (_i32, [_vp, _u32, _u32, _vp, _i32, _i32, _u64, _u64, _vp]),
    "ngp_mip_resample": (_i32, [_vp, _u32, _u32, _vp, _vp, _f32, _i32, _u64, _u64, _vp]),
    "ngp_mip_encode": (_i32, [_vp, _u32, _u32, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "ngp_mip_rays_multi": (_i32, [_vp, _u32, _vp, _u32, _vp, _vp, _vp, _f32, _i32, _vp, _i32, _vp, _vp, _vp]),
    "ngp_mip_encode_deg": (_i32, [_vp, _u32, _u32, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "ngp_mip_param_count": (_i32, [_i32, _vp]),
    "ngp_mip_workspace_bytes": (_i32, [_i32, _u32, _vp, _vp]),
    "ngp_mip_fwd_deg": (_i32, [_vp, _u32, _u32, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "ngp_mip_bwd_deg": (_i32, [_vp, _u32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "ngp_mip_fwd": (_i32, [_vp, _u32, _u32, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "ngp_mip_composite_fwd": (_i32, [_vp, _u32, _u32, _vp, _i32, _vp, _vp, _f32, _f32, _i32, _vp, _vp, _vp, _vp]),
    "ngp_mip_composite_loss_bwd": (_i32, [_vp, _u32, _u32, _vp, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _i32, _f32, _f32, _vp, _vp, _vp]),
    "ngp_pixelnerf_param_count": (_i32, [_vp]),
    "ngp_pixelnerf_workspace_bytes": (_i32, [_u32, _u32, _vp, _vp, _vp]),
    "ngp_pixelnerf_fwd": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _vp, _f32, _i32, _vp, _vp, _vp]),
    "ngp_pixelnerf_bwd": (_i32, [_vp, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_pixelnerf_composite_fwd": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_pixelnerf_composite_loss_bwd": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp]),
    "ngp_svox_train_step": (_i32, [_vp, _u32, _vp, _u32, _u32, _vp, _f32, _f32, _f32, _f32, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _vp]),
    "ngp_svox_render": (_i32, [_vp, _u32, _u32, _u32, _vp, _f32, _f32, _f32, _f32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "ngp_svox_tv_grad": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _u32, _u32, _u32, _f32, _i32, _vp, _vp]),
    "ngp_svox_rmsprop": (_i32, [_vp, _u64, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32]),
    "ngp_svox_sample": (_i32, [_vp, _u32, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _vp]),
    "ngp_svox_weight_render": (_i32, [_vp, _u32, _u32, _vp, _f32, _f32, _f32, _f32, _vp, _i32, _i32, _i32, _vp, _f32, _f32, _vp]),
    "ngp_svox_dilate": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "ngp_svox_compact_workspace_bytes": (_i32, [_i32, _i32, _i32, _vp]),
    "ngp_svox_compact": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "ngp_mesh_workspace_bytes": (_i32, [_u32, _u64, _u64, _vp]),
    "ngp_density_lattice": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp]),
    "ngp_marching_cubes": (_i32, [_vp, _u32, _vp, _f32, _vp, _vp, _u64, _vp, _u64, _vp]),
    "ngp_mesh_largest_component": (_i32, [_vp, _u64, _u64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_mesh_vertex_normals": (_i32, [_vp, _u64, _u64, _vp, _vp, _vp, _vp]),
    "ngp_mesh_smooth_workspace_bytes": (_i32, [_u32, _u32, _vp]),
    "ngp_mesh_smooth": (_i32, [_vp, _u32, _vp, _u32, _u32, _vp, _u64, _vp, _vp]),
    "ngp_render_workspace_bytes": (_i32, [_u32, _u32, _vp]),
    "ngp_render_init": (_i32, [_vp, _u32, _u32, _vp, _f32, _f32, _vp, _vp, _f32, _f32, _u32, _i32, _u64, _u64, _u32, _vp, _vp, _vp, _vp]),
    "ngp_render_march_round": (_i32, [_vp, _u32, _u32, _vp, _u32, _u32, _f32, _f32, _vp, _vp, _vp, _f32, _u32, _i32]),
    "ngp_render_composite_round": (_i32, [_vp, _u32, _u32, _vp, _u32, _u32, _f32, _u32, _vp, _vp, _vp, _vp]),
    "ngp_march_workspace_bytes": (_u64, [_u32]),
    "ngp_march": (_i32, [_vp, _u32, _f32, _f32, _u32, _vp, _vp, _vp, _f32, _f32, _u32, _i32, _u64, _u64, _vp, _vp, _vp, _vp, _vp]),
    "ngp_compact": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _i32]),
    "ngp_composite_fwd": (_i32, [_vp, _u32, _vp, _i32, _vp, _vp, _vp, _vp, _u32, _vp]),
    "ngp_composite_bwd": (_i32, [_vp, _u32, _u32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _u32, _vp]),
    "ngp_composite_infer": (_i32, [_vp, _u32, _vp, _i32, _vp, _vp, _u32, _vp, _vp]),
    "ngp_composite_loss_bwd": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _vp, _u32, _vp, _vp, _vp, _f32]),
    "ngp_grid_mark_untrained": (_i32, [_vp, _u32, _vp, _u32, _vp, _vp, _i32, _i32]),
    "ngp_grid_generate_samples": (_i32, [_vp, _u32, _u64, _u64, _vp, _f32, _f32, _vp, _vp, _vp, _u32, _f32]),
    "ngp_grid_splat": (_i32, [_vp, _u32, _vp, _vp, _i32, _vp]),
    "ngp_grid_ema": (_i32, [_vp, _u32, _f32, _vp, _vp]),
    "ngp_grid_update_bitfield": (_i32, [_vp, _vp, _vp, _vp, _u32]),
    "ngp_adam_ema": (_i32, [_vp, _u64, _vp, _i32, _vp, _i32, _f32, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _u32, _f32, _i32]),
    "ngp_train_sweep": (_i32, [_vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _u32,
                               _f32]),
    "ngp_dp_exchange_step": (_i32, [_vp, _i32, _i32, _u64, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32,
                                    _f32, _f32, _u32, _f32]),
    "ngp_dp_exchange_wait": (_i32, [_vp, _i32, _vp, _u32]),
    "ngp_ipc_export": (_i32, [_vp, _vp, _vp]),
    "ngp_ipc_open": (_i32, [_vp, _u64, _vp]),
    "ngp_ipc_close": (_i32, [_vp, _u64]),
    "ngp_raygen": (_i32, [_vp, _u32, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ngp_prepare_batch": (_i32, [_vp, _u32, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "ngp_blend_target": (_i32, [_vp, _u32, _vp, _vp, _vp]),
    "ngp_pcg32_seed": (None, [_u64, _u64, _vp]),
    "ngp_pcg32_advance": (None, [_vp, _i64]),
}

# kernels launched by each entry point (our own __global__ functions; memsets not counted) -- bench.py's gpu_launches
KERNELS_PER_CALL = {
    "ngp_hash_level_table": 1, "ngp_hash_level_table_primes": 1, "ngp_hash_fwd": 1, "ngp_hash_bwd": 1, "ngp_sh_fwd": 1, "ngp_mlp_fwd": 1, "ngp_mlp_bwd": 1, "ngp_mlp_bwd_dgrad": 1,
    "ngp_network_fwd": 1, "ngp_network_bwd": 1, "ngp_network_bwd_fx": 1, "ngp_train_sweep": 1, "ngp_density_fwd": 1, "ngp_march": 3, "ngp_compact": 1, "ngp_composite_fwd": 1,
    "ngp_composite_bwd": 1, "ngp_composite_infer": 1, "ngp_composite_loss_bwd": 1, "ngp_grid_mark_untrained": 1,
    "ngp_grid_generate_samples": 1, "ngp_grid_splat": 1, "ngp_grid_ema": 1, "ngp_grid_update_bitfield": 7, "ngp_adam_ema": 1, "ngp_dp_exchange_step": 1, "ngp_dp_exchange_wait": 1, "ngp_raygen": 1, "ngp_prepare_batch": 1,
    "ngp_blend_target": 1,
    "ngp_density_lattice": 1, "ngp_marching_cubes": 3, "ngp_mesh_largest_component": 18, "ngp_mesh_vertex_normals": 7,
    "ngp_render_init": 3, "ngp_render_march_round": 3, "ngp_render_composite_round": 3,
    "ngp_nerf_fwd": 1, "ngp_nerf_density": 1, "ngp_nerf_bwd": 3,
    "ngp_mip_rays": 1, "ngp_mip_sample": 1, "ngp_mip_resample": 1, "ngp_mip_encode": 1, "ngp_mip_fwd": 1, "ngp_mip_composite_fwd": 1,
    "ngp_mip_composite_loss_bwd": 1, "ngp_mip_rays_multi": 1, "ngp_mip_encode_deg": 1, "ngp_mip_fwd_deg": 1,
    "ngp_mip_bwd_deg": 3,
    "ngp_pixelnerf_fwd": 18, "ngp_pixelnerf_bwd": 74, "ngp_pixelnerf_composite_fwd": 1, "ngp_pixelnerf_composite_loss_bwd": 1,
    "ngp_svox_train_step": 1, "ngp_svox_render": 1, "ngp_svox_tv_grad": 1, "ngp_svox_rmsprop": 1, "ngp_svox_sample": 1, "ngp_svox_weight_render": 1,
    "ngp_svox_dilate": 1, "ngp_svox_compact": 5,
}
launch_count = 0
_lib = None


class NgpError(RuntimeError):
    pass


def load():
    """dlopen the in-tree library; raises if it has not been built (python -m jnerf_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NgpError(f"{LIB_PATH} is missing: build it with `python jnerf_b200/build.py` (nvcc, sm_90a). "
                           "There is no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError here = header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def call(name, *args):
    """Call an int-returning entry point and raise NgpError(ngp_last_error()) on a non-zero status."""
    global launch_count
    lib = load()
    launch_count += KERNELS_PER_CALL.get(name, 0)
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise NgpError(f"{name} failed ({rc}): {lib.ngp_last_error().decode()}")
    return rc
