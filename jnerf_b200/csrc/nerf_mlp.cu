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
// ---- backward 1: the dgrad chain of one tile, every layer's dY into the scratch ----------------------------------------------------
__global__ void __launch_bounds__(THREADS, 1)
    nerf_dgrad_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ P, const __half* __restrict__ saved,
                      const __half* __restrict__ dout, __half* __restrict__ dys) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Ga = smem;                     // 32 groups
    uint8_t* Gb = Ga + 32 * GB;             // 34 groups: dY of kernel layer 8 = [dalpha, 0 x 15, df]
    uint8_t* S = Gb + 34 * GB;              // 2 groups: dY of rgb_linear = [drgb, 0 x 13]
    uint8_t* W0 = S + 2 * GB;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t row0 = blockIdx.x * ROWS;
    if (row0 >= n) return;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u;
    const __half* sv = saved + (size_t)blockIdx.x * S_GROUPS * ROWS * 8;
    __half* dy = dys + (size_t)blockIdx.x * D_GROUPS * ROWS * 8;
    Pipe pipe{{W0, W0 + BWD_WBUF}, 0, BWD_CHUNKS, P, true};
    stage(W0, bwd_chunk(P, 0), tid);
    for (uint32_t t = tid; t < ROWS; t += THREADS) {
        uint2 v = make_uint2(0u, 0u);
        if (row0 + t < n) v = __ldg(reinterpret_cast<const uint2*>(dout) + row0 + t);
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        const uint4 rgb = make_uint4(v.x, v.y & 0xFFFFu, 0u, 0u), alpha = make_uint4(v.y >> 16, 0u, 0u, 0u);
        auto at = [&](uint8_t* base, uint32_t g) { return reinterpret_cast<uint4*>(base + g * GB + t * 16); };
        *at(S, 0) = rgb;
        *at(S, 1) = z;
        *at(Gb, 0) = alpha;
        *at(Gb, 1) = z;
        uint8_t* d8 = reinterpret_cast<uint8_t*>(dy);
        *at(d8, D_10) = rgb;
        for (uint32_t g = 1; g < 8; ++g) *at(d8, D_10 + g) = z;
        *at(d8, D_8) = alpha;
        *at(d8, D_8 + 1) = z;
        for (uint32_t g = 34; g < 40; ++g) *at(d8, D_8 + g) = z;
    }
    auto kmaj = [&](const uint8_t* s, uint32_t kb) { return slab_desc_kmajor(smem_u32(s) + m * 64 * 16, ROWS, 0, kb); };
    // rgb_linear: dY10 (K = 16) -> dY9 = dv * ReLU'(v)
#pragma unroll 1
    for (uint32_t j = 0; j < 2; ++j) {
        const uint32_t w = pipe.begin(tid);
        float d[32];
        gemm_bwd<64, 16>(d, [&](uint32_t kb) { return kmaj(S, kb); }, w);
        epi_bwd<true>(d, sv, S_V + 8 * j, Ga, 8 * j, dy, D_9 + 8 * j, m, tw);
        pipe.end();
    }
    // views_linears.0: dY9 (K = 128) -> df (feature_linear has no activation), after [dalpha, 0]
#pragma unroll 1
    for (uint32_t j = 0; j < 4; ++j) {
        const uint32_t w = pipe.begin(tid);
        float d[32];
        gemm_bwd<64, 128>(d, [&](uint32_t kb) { return kmaj(Ga, kb); }, w);
        epi_bwd<false>(d, sv, 0, Gb, 2 + 8 * j, dy, D_8 + 2 + 8 * j, m, tw);
        pipe.end();
    }
    // alpha_linear + feature_linear: dY8 (K = 272) -> dY7 = dh7 * ReLU'(h7)
#pragma unroll 1
    for (uint32_t j = 0; j < 4; ++j) {
        const uint32_t w = pipe.begin(tid);
        float d[32];
        gemm_bwd<64, 272>(d, [&](uint32_t kb) { return kmaj(Gb, kb); }, w);
        epi_bwd<true>(d, sv, S_H + 32 * 7 + 8 * j, Ga, 8 * j, dy, D_H + 32 * 7 + 8 * j, m, tw);
        pipe.end();
    }
    // pts_linears.7 .. 1: dY_l -> dY_{l-1} (layer 5: the h4 columns of its concatenated input only)
#pragma unroll 1
    for (uint32_t l = 7; l >= 1; --l) {
        const uint8_t* src = (l & 1) ? Ga : Gb;
        uint8_t* dst = (l & 1) ? Gb : Ga;
#pragma unroll 1
        for (uint32_t j = 0; j < 4; ++j) {
            const uint32_t w = pipe.begin(tid);
            float d[32];
            gemm_bwd<64, 256>(d, [&](uint32_t kb) { return kmaj(src, kb); }, w);
            epi_bwd<true>(d, sv, S_H + 32 * (l - 1) + 8 * j, dst, 8 * j, dy, D_H + 32 * (l - 1) + 8 * j, m, tw);
            pipe.end();
        }
    }
}

// ---- backward 2: weight and bias gradients, dW_l = sum over rows of dY_l^T X_l, per row chunk --------------------------------------
// A job is (layer, 64 output rows, 128 input columns); warpgroup m takes input columns [64m, 64m+64) of it.  Chunk c of NCHUNK
// covers tiles [c T / NCHUNK, (c+1) T / NCHUNK) and writes its sums (plain stores, every parameter exactly once) to part[c].
constexpr uint32_t n_jobs() {
    uint32_t s = 0;
    for (uint32_t l = 0; l < NL; ++l) s += (out_pad(l) + 63) / 64 * ((in_pad(l) + 127) / 128);
    return s;
}
constexpr uint32_t WGRAD_JOBS = n_jobs();
__device__ __forceinline__ uint32_t dy_base(uint32_t l) { return l < 8 ? D_H + 32 * l : l == 8 ? D_8 : l == 9 ? D_9 : D_10; }
// saved group holding input column `col` of layer l
__device__ __forceinline__ uint32_t x_group(uint32_t l, uint32_t col) {
    if (l == 0) return S_ENC + col / 8;
    if (l == 5) return col < 64 ? S_ENC + col / 8 : S_H + 32 * 4 + (col - 64) / 8;
    if (l == 9) return col < 256 ? S_F + col / 8 : S_DIR + (col - 256) / 8;
    if (l == 10) return S_V + col / 8;
    return S_H + 32 * (l - 1) + col / 8;
}

__global__ void __launch_bounds__(THREADS, 2)
    nerf_wgrad_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ saved, const __half* __restrict__ dys,
                      float* __restrict__ part) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* A[2] = {smem, smem + 8 * GB};
    uint8_t* B[2] = {smem + 16 * GB, smem + 32 * GB};
    uint32_t idx = blockIdx.x, l = 0;
    for (;; ++l) {
        const uint32_t nj = (out_pad(l) + 63) / 64 * ((in_pad(l) + 127) / 128);
        if (idx < nj) break;
        idx -= nj;
    }
    const uint32_t nib = (in_pad(l) + 127) / 128, ob = idx / nib, ib = idx % nib;
    const uint32_t in = in_pad(l), outp = out_pad(l), c = blockIdx.y;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u, col_wg = 128 * ib + 64 * m;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t T = (n + ROWS - 1) / ROWS, t0 = (uint32_t)((uint64_t)c * T / NCHUNK), t1 = (uint32_t)((uint64_t)(c + 1) * T / NCHUNK);
    auto stage_tile = [&](uint32_t t, uint32_t b) {
        const __half* a_src = dys + ((size_t)t * D_GROUPS + dy_base(l) + 8 * ob) * ROWS * 8;
        for (uint32_t i = tid; i < 8 * ROWS; i += THREADS) cp_async16(smem_u32(A[b]) + i * 16, a_src + (size_t)i * 8);
        for (uint32_t i = tid; i < 16 * ROWS; i += THREADS) {
            const uint32_t col = 128 * ib + 8 * (i / ROWS);
            if (col < in) cp_async16(smem_u32(B[b]) + i * 16, saved + ((size_t)t * S_GROUPS + x_group(l, col)) * ROWS * 8 + (i % ROWS) * 8);
        }
        cp_async_commit();
    };
    const bool bias_thread = ib == 0 && m == 0 && tw < 64;
    const bool active = col_wg < in;
    float d[32];
#pragma unroll
    for (uint32_t i = 0; i < 32; ++i) d[i] = 0.f;
    float bsum = 0.f;
    if (t0 < t1) stage_tile(t0, 0);
#pragma unroll 1
    for (uint32_t t = t0; t < t1; ++t) {
        cp_async_wait_all();
        fence_proxy_async_smem();
        __syncthreads();
        if (t + 1 < t1) stage_tile(t + 1, (t + 1 - t0) & 1);
        const uint32_t b = (t - t0) & 1;
        // a warpgroup past the layer's last input column multiplies unstaged columns and discards them: no branch around the wgmmas,
        // which the compiler would otherwise serialise
        wgmma_fence();
        mlp::mma_wgrad<64>(d, smem_u32(A[b]), 0, smem_u32(B[b]), 8 * m, 1u);
        wgmma_commit();
        if (bias_thread) {
            const uint8_t* col = A[b] + (tw / 8) * GB + (tw % 8) * 2;
#pragma unroll 8
            for (uint32_t r = 0; r < ROWS; ++r) bsum += __half2float(*reinterpret_cast<const __half*>(col + r * 16));
        }
        wgmma_wait<0>();
    }
    float* dst = part + (size_t)c * N_PARAMS;
    if (active) {
        const uint32_t r0 = frag_row(tw), c0 = 2 * (tw & 3u);
#pragma unroll
        for (uint32_t cc = 0; cc < 8; ++cc)
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
                for (uint32_t j = 0; j < 2; ++j) {
                    const uint32_t orow = 64 * ob + r0 + 8 * h, icol = col_wg + 8 * cc + c0 + j;
                    if (orow < outp && icol < in) dst[w_off(l) + orow * in + icol] = d[4 * cc + 2 * h + j];
                }
    }
    if (bias_thread && 64 * ob + tw < outp) dst[b_off(l) + 64 * ob + tw] = bsum;
}

__global__ void nerf_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ grad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N_PARAMS) return;
    float s = part[i];
#pragma unroll
    for (uint32_t c = 1; c < NCHUNK; ++c) s += part[(size_t)c * N_PARAMS + i];
    grad[i] = s;
}

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
