// oracle/_ref build: the reference's Plenoxels render kernels (contrib/plenoxel volume_render_cuvol_fused.h) compiled UNMODIFIED
// for sm_90a where they lie, behind extern "C" launchers with volume_render_cuvol.py's launch shapes and the RenderOptions defaults
// the reference's runner uses.  TEST / BENCH INFRASTRUCTURE: never linked into libngp_b200.so.
#include "volume_render_cuvol_fused.h"

namespace {
jittor::Var var(const void* p, int64_t a, int64_t b = 1, int64_t c = 1) {
    jittor::Var v{const_cast<void*>(p), {a, b, c, 1}, a * b * c};
    return v;
}
const RenderOptions OPT{1.0f, 0.5f, 1e-10f, 1e-7f, 0.0f, false, false};
}  // namespace

// Q rays (origins, unit dirs (Q, 3)) through a grid of links (X, Y, Z), density (cap, 1), sh (cap, 27); offset / scaling (3,) device
// arrays in grid units (_offset * reso - 0.5, _scaling * reso).  ref_svox_render: out (Q, 3).  ref_svox_backward: the gradient of the
// MSE against gt (Q, 3) given the forward's rgb (grad_out_is_rgb), added into grad_density (cap,) / grad_sh (cap, 27) with float atomics.
extern "C" int ref_svox_render(int Q, const float* origins, const float* dirs, const int32_t* links, int X, int Y, int Z, int cap,
                               const float* density, const float* sh, const float* offset, const float* scaling, float* out, void* stream) {
    jittor::Var d = var(density, cap, 1), s = var(sh, cap, 27), l = var(links, X, Y, Z), off = var(offset, 3), scl = var(scaling, 3);
    jittor::Var empty = var(nullptr, 0), o = var(origins, Q, 3), di = var(dirs, Q, 3), res = var(out, Q, 3);
    empty.num = 0;
    PackedSparseGridSpec grid(&d, &s, &l, &off, &scl, &empty, &empty, 9, 1, &empty);
    const int blocks = CUDA_N_BLOCKS_NEEDED(Q * WARP_SIZE, TRACE_RAY_CUDA_THREADS);
    render_ray_kernel<<<blocks, TRACE_RAY_CUDA_THREADS, 0, (cudaStream_t)stream>>>(grid, PackedRaysSpec(&o, &di), OPT, PackedVar32<float, 2>(&res), nullptr);
    return (int)cudaGetLastError();
}

extern "C" int ref_svox_backward(int Q, const float* origins, const float* dirs, const int32_t* links, int X, int Y, int Z, int cap,
                                 const float* density, const float* sh, const float* offset, const float* scaling, const float* gt,
                                 const float* rgb, float* grad_density, float* grad_sh, void* stream) {
    jittor::Var d = var(density, cap, 1), s = var(sh, cap, 27), l = var(links, X, Y, Z), off = var(offset, 3), scl = var(scaling, 3);
    jittor::Var empty = var(nullptr, 0), o = var(origins, Q, 3), di = var(dirs, Q, 3), gd = var(grad_density, cap, 1), gs = var(grad_sh, cap, 27);
    empty.num = 0;
    PackedSparseGridSpec grid(&d, &s, &l, &off, &scl, &empty, &empty, 9, 1, &empty);
    PackedGridOutputGrads grads(&gd, &gs, &empty, &empty);
    const int blocks = CUDA_N_BLOCKS_NEEDED(Q * WARP_SIZE, TRACE_RAY_CUDA_THREADS);
    render_ray_backward_kernel<<<blocks, TRACE_RAY_CUDA_THREADS, 0, (cudaStream_t)stream>>>(grid, gt, rgb, PackedRaysSpec(&o, &di), OPT, true,
                                                                                            nullptr, 0.f, 0.f, grads, nullptr, nullptr);
    return (int)cudaGetLastError();
}
