// MipNerfMLP at 16 IPE degrees (multicam.py: max_deg_point = 16) on the kernels of nerf_mlp.cuh at 12 encoder groups: the 96 IPE columns
// feed pts_linears.0 (in_pad 96) and the skip layer (in_pad 352, streamed as two K-chunks), the other layers are section 10's.  Forward,
// dgrad, wgrad and the chunk-ordered reduce; the saved block is 320 groups.  Built with -fmad=false, like mip_multiscale.cu's fp32 encoder:
// the encode stage forms the same IPE bit for bit before its fp16 rounding (at degree 15 one contracted multiply-add in mip::gaussian moves
// a column by ~1e-2).  DESIGN.md section 11.
#include "mip_common.cuh"
#include "nerf_mlp.cuh"

namespace nerf {
constexpr uint32_t WIDE_DEGS = 16, WIDE_EG = 6 * WIDE_DEGS / 8;
using WL = Layout<WIDE_EG>;

// MipEnc of mip_mlp.cu at 16 degrees: the 96 IPE columns [sin | cos], deg-major, xyz inner, fill the 12 groups exactly.
struct MipEncWide {
    static constexpr uint32_t EG = WIDE_EG;
    const float* t;
    uint32_t cylinder, integrate;
    int min_deg;
    __device__ __forceinline__ void pos(uint8_t* slab, const float* rays, uint32_t S, uint32_t row0, uint32_t n, uint32_t tid) const {
        for (uint32_t k = tid; k < ROWS * 3; k += THREADS) {
            const uint32_t r = k / 3, dim = k % 3, row = row0 + r;
            auto put = [&](uint32_t f, float v) { *reinterpret_cast<__half*>(slab + (f / 8) * GB + r * 16 + (f % 8) * 2) = __float2half_rn(v); };
            float mean = 0.f, var = 0.f;
            if (row < n) {
                const uint32_t ray = row / S, i = row % S;
                const float* tt = t + (size_t)ray * (S + 1) + i;
                mip::gaussian(rays + (size_t)ray * mip::RAY_FLOATS, tt[0], tt[1], dim, cylinder, integrate, mean, var);
            }
            mip::ipe<WIDE_DEGS>(mean, var, dim, min_deg, put);
        }
    }
    __device__ __forceinline__ void dir(uint8_t* slab, const float* rays, uint32_t S, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<mip::VIEW_DEGS>(slab, [&](uint32_t row, uint32_t dim) { return rays[(size_t)(row / S) * mip::RAY_FLOATS + 6 + dim]; }, row0, n, tid);
    }
};

__global__ void __launch_bounds__(THREADS, 1)
    mip_wide_dgrad_kernel(uint32_t n_max, const __half* __restrict__ P, const __half* __restrict__ saved, const __half* __restrict__ dout,
                          __half* __restrict__ dys) {
    dgrad_body<WIDE_EG>(n_max, nullptr, P, saved, dout, dys);
}
__global__ void __launch_bounds__(THREADS, 2)
    mip_wide_wgrad_kernel(uint32_t n_max, const __half* __restrict__ saved, const __half* __restrict__ dys, float* __restrict__ part) {
    wgrad_body<WIDE_EG>(n_max, nullptr, saved, dys, part);
}
__global__ void mip_wide_reduce_kernel(const float* __restrict__ part, float* __restrict__ grad) { wgrad_reduce_body<WIDE_EG>(part, grad); }
}  // namespace nerf

using namespace nerf;

extern "C" {

int ngp_mip_param_count(int degs, uint64_t* count_out) {
    NGP_REQUIRE(degs == 8 || degs == 16, "ngp_mip_param_count: degs must be 8 or 16");
    *count_out = degs == 8 ? N_PARAMS : WL::N_PARAMS;
    return 0;
}

int ngp_mip_workspace_bytes(int degs, uint32_t n_max, uint64_t* saved_bytes, uint64_t* scratch_bytes) {
    NGP_REQUIRE(degs == 8 || degs == 16, "ngp_mip_workspace_bytes: degs must be 8 or 16");
    if (degs == 8) return ngp_nerf_workspace_bytes(n_max, saved_bytes, scratch_bytes);
    *saved_bytes = tiles(n_max) * WL::S_GROUPS * GB;
    *scratch_bytes = tiles(n_max) * D_GROUPS * GB + (uint64_t)NCHUNK * WL::N_PARAMS * 4;
    return 0;
}

int ngp_mip_fwd_deg(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate,
                    int min_deg, int degs, const void* params, void* out, void* saved) {
    NGP_REQUIRE(degs == 8 || degs == 16, "ngp_mip_fwd_deg: degs must be 8 or 16");
    if (degs == 8) return ngp_mip_fwd(stream, n_rays, n_samples, rays, t, ray_shape, integrate, min_deg, params, out, saved);
    NGP_REQUIRE(n_samples > 0 && (uint64_t)n_rays * n_samples < (1ull << 32), "ngp_mip_fwd_deg: n_samples must be > 0 and n_rays * n_samples < 2^32");
    NGP_REQUIRE(ray_shape == 0 || ray_shape == 1, "ngp_mip_fwd_deg: ray_shape must be 0 (cone) or 1 (cylinder)");
    const uint32_t n = n_rays * n_samples;
    if (n == 0) return 0;
    NGP_REQUIRE(rays && t && params && out, "ngp_mip_fwd_deg: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)saved & 15) == 0, "ngp_mip_fwd_deg: params / saved must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const MipEncWide enc{t, (uint32_t)ray_shape, (uint32_t)(integrate != 0), min_deg};
    return saved ? launch_fwd<false, true>(s, n, nullptr, rays, n_samples, params, out, saved, enc)
                 : launch_fwd<false, false>(s, n, nullptr, rays, n_samples, params, out, nullptr, enc);
}

int ngp_mip_bwd_deg(void* stream, uint32_t n_max, int degs, const void* params, const void* saved, const void* dout, void* scratch, float* grad) {
    NGP_REQUIRE(degs == 8 || degs == 16, "ngp_mip_bwd_deg: degs must be 8 or 16");
    if (degs == 8) return ngp_nerf_bwd(stream, n_max, nullptr, params, saved, dout, scratch, grad);
    NGP_REQUIRE(params && grad && scratch && (n_max == 0 || (saved && dout)), "ngp_mip_bwd_deg: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)saved & 15) == 0 && ((uintptr_t)scratch & 15) == 0 && ((uintptr_t)dout & 7) == 0,
                "ngp_mip_bwd_deg: misaligned buffer");
    cudaStream_t s = (cudaStream_t)stream;
    __half* dys = (__half*)scratch;
    float* part = (float*)((uint8_t*)scratch + tiles(n_max) * D_GROUPS * GB);
    if (n_max > 0) {
        if (ngp_first_use((const void*)mip_wide_dgrad_kernel))
            NGP_CHECK_CUDA(cudaFuncSetAttribute(mip_wide_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
        mip_wide_dgrad_kernel<<<(uint32_t)tiles(n_max), THREADS, BWD_SMEM, s>>>(n_max, (const __half*)params, (const __half*)saved,
                                                                               (const __half*)dout, dys);
        NGP_LAUNCH_CHECK();
    }
    if (ngp_first_use((const void*)mip_wide_wgrad_kernel))
        NGP_CHECK_CUDA(cudaFuncSetAttribute(mip_wide_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGRAD_SMEM));
    mip_wide_wgrad_kernel<<<dim3(n_jobs(WIDE_EG), NCHUNK), THREADS, WGRAD_SMEM, s>>>(n_max, (const __half*)saved, dys, part);
    NGP_LAUNCH_CHECK();
    mip_wide_reduce_kernel<<<(WL::N_PARAMS + 255) / 256, 256, 0, s>>>(part, grad);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
