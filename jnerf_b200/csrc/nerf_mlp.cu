// Vanilla NeRF network (models/networks/ori_nerf_network.py + position_encoders/freq_encoder/freq_encoder.py of the reference) on
// Hopper wgmma: the frequency encoding and the 8x256 trunk with its skip, alpha / feature / views / rgb heads.  DESIGN.md section 10.
//
// Parameters: ONE flat fp16 vector, per kernel layer l the weight (out_pad(l), in_pad(l)) row-major, then the bias (out_pad(l)).
// Padding rows / columns are zero and receive zero gradient.  Kernel layer 8 is alpha_linear (row 0 of 16) stacked on feature_linear
// (rows 16..271): both read h7, and alpha first lets the density kernel stop after one 16-row chunk.
//
// A CTA is two warpgroups on a 128-row tile, warpgroup m owning rows [64m, 64m+64) of every activation slab (wgmma.cuh); the weights
// do not fit in shared memory (1.2 MB), so they stream through two cp.async buffers in chunks of 64 output rows (forward) or 64 input
// columns (dgrad), the next chunk loading while the current one multiplies.
#include "nerf_mlp.cuh"

namespace nerf {
// ---- backward 1: the dgrad chain of one tile, every layer's dY into the scratch (dgrad_body, nerf_mlp.cuh) ----------------------------
__global__ void __launch_bounds__(THREADS, 1)
    nerf_dgrad_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ P, const __half* __restrict__ saved,
                      const __half* __restrict__ dout, __half* __restrict__ dys) {
    dgrad_body<8>(n_max, n_dev, P, saved, dout, dys);
}

// ---- backward 2: weight and bias gradients per row chunk (wgrad_body), summed in chunk order (wgrad_reduce_body) ------------------------
__global__ void __launch_bounds__(THREADS, 2)
    nerf_wgrad_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ saved, const __half* __restrict__ dys,
                      float* __restrict__ part) {
    wgrad_body<8>(n_max, n_dev, saved, dys, part);
}

__global__ void nerf_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ grad) { wgrad_reduce_body<8>(part, grad); }

}  // namespace nerf

using namespace nerf;

extern "C" {

int ngp_nerf_param_count(uint64_t* count_out) {
    *count_out = N_PARAMS;
    return 0;
}

int ngp_nerf_workspace_bytes(uint32_t n_max, uint64_t* saved_bytes, uint64_t* scratch_bytes) {
    *saved_bytes = tiles(n_max) * S_GROUPS * GB;
    *scratch_bytes = tiles(n_max) * D_GROUPS * GB + (uint64_t)NCHUNK * N_PARAMS * 4;
    return 0;
}

int ngp_nerf_fwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* params, void* out, void* saved) {
    if (n_max == 0) return 0;
    NGP_REQUIRE(coords && params && out, "ngp_nerf_fwd: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)saved & 15) == 0, "ngp_nerf_fwd: params / saved must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    return saved ? launch_fwd<false, true>(s, n_max, n_dev, coords, 7, params, out, saved)
                 : launch_fwd<false, false>(s, n_max, n_dev, coords, 7, params, out, nullptr);
}

int ngp_nerf_density(void* stream, uint32_t n, const float* pos, const void* params, void* sigma_out) {
    if (n == 0) return 0;
    NGP_REQUIRE(pos && params && sigma_out, "ngp_nerf_density: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0, "ngp_nerf_density: params must be 16-byte aligned");
    return launch_fwd<true, false>((cudaStream_t)stream, n, nullptr, pos, 3, params, sigma_out, nullptr);
}

int ngp_nerf_bwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const void* params, const void* saved, const void* dout, void* scratch,
                 float* grad) {
    NGP_REQUIRE(params && grad && scratch && (n_max == 0 || (saved && dout)), "ngp_nerf_bwd: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)saved & 15) == 0 && ((uintptr_t)scratch & 15) == 0 && ((uintptr_t)dout & 7) == 0,
                "ngp_nerf_bwd: misaligned buffer");
    cudaStream_t s = (cudaStream_t)stream;
    __half* dys = (__half*)scratch;
    float* part = (float*)((uint8_t*)scratch + tiles(n_max) * D_GROUPS * GB);
    if (n_max > 0) {
        if (ngp_first_use((const void*)nerf_dgrad_kernel))
            NGP_CHECK_CUDA(cudaFuncSetAttribute(nerf_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
        nerf_dgrad_kernel<<<(uint32_t)tiles(n_max), THREADS, BWD_SMEM, s>>>(n_max, n_dev, (const __half*)params, (const __half*)saved,
                                                                          (const __half*)dout, dys);
        NGP_LAUNCH_CHECK();
    }
    if (ngp_first_use((const void*)nerf_wgrad_kernel))
        NGP_CHECK_CUDA(cudaFuncSetAttribute(nerf_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGRAD_SMEM));
    nerf_wgrad_kernel<<<dim3(WGRAD_JOBS, NCHUNK), THREADS, WGRAD_SMEM, s>>>(n_max, n_dev, (const __half*)saved, dys, part);
    NGP_LAUNCH_CHECK();
    nerf_wgrad_reduce_kernel<<<(N_PARAMS + 255) / 256, 256, 0, s>>>(part, grad);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
