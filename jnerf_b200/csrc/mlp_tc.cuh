// Building blocks of the fully-fused MLP on Hopper wgmma (used by mlp_tc.cu and fused_net.cu).
// A tile is 128 rows (samples), processed by one warpgroup; loads and global copies use "thread t = row t", epilogues the wgmma
// accumulator fragment.  Activations and gradients live in shared-memory "slabs" (see wgmma.cuh) and never leave the SM between layers.
#pragma once
#include "wgmma.cuh"
#include "ngp_common.cuh"

namespace mlp {
using namespace wg;

constexpr uint32_t ROWS = 128;
constexpr uint32_t GB = ROWS * 16;          // bytes of one slab feature-group (8 features x 128 rows)

// ---- weights: global (out=rows, in=K) row-major  ->  smem [K/8][rows][8] (canonical K-major B operand) ----
// Inlined form for kernels that move registers between warpgroups (setmaxnreg): ptxas applies the per-warpgroup counts only to a
// kernel without calls, and otherwise compiles every warpgroup at the launch count.
__device__ __forceinline__ void stage_weights_inline(uint8_t* dst, const __half* __restrict__ W, int rows, int K, int tid, int nthr) {
    const int kg = K / 8;
    for (int i = tid; i < rows * kg; i += nthr) {
        const int n = i / kg, g = i % kg;
        *reinterpret_cast<uint4*>(dst + (size_t)g * rows * 16 + n * 16) = __ldg(reinterpret_cast<const uint4*>(W + (size_t)n * K + g * 8));
    }
}
static __device__ __noinline__ void stage_weights(uint8_t* dst, const __half* __restrict__ W, int rows, int K, int tid, int nthr) {
    stage_weights_inline(dst, W, rows, K, tid, nthr);
}

// ---- MMA issue (all 128 threads of one warpgroup) ----------------------------------------------------------
// A 128-row tile is two wgmma row blocks: m = 0 covers rows [0, 64), m = 1 rows [64, 128).  Every shape is a template parameter and
// every shared-memory offset a value of the kernel, so the K loop unrolls into back-to-back wgmmas.
//
// D[64 x N] = rows [64m, 64m+64) of ACT[:, 8*g0 .. 8*g0+K) * W^T          (W staged with rows = N)
template <uint32_t K, uint32_t N>
__device__ __forceinline__ void mma_fwd(float (&d)[N / 2], uint32_t act_s, uint32_t g0, uint32_t w_s, uint32_t m) {
#pragma unroll
    for (uint32_t kb = 0; kb < K / 16; ++kb)
        mma<N, 0, 0>(d, slab_desc_kmajor(act_s + m * 64 * 16, ROWS, g0, kb), slab_desc_kmajor(w_s, N, 0, kb), kb > 0 ? 1u : 0u);
}
// D[64 x NIN] = rows [64m, 64m+64) of GRD[:, 8*g0 .. 8*g0+KOUT) * W[:, 0..NIN)          (W staged with rows = KOUT; read MN-major)
template <uint32_t KOUT, uint32_t NIN>
__device__ __forceinline__ void mma_dgrad(float (&d)[NIN / 2], uint32_t grd_s, uint32_t g0, uint32_t w_s, uint32_t m) {
#pragma unroll
    for (uint32_t kb = 0; kb < KOUT / 16; ++kb)
        mma<NIN, 0, 1>(d, slab_desc_kmajor(grd_s + m * 64 * 16, ROWS, g0, kb), slab_desc_mnmajor(w_s, KOUT, 0, kb), kb > 0 ? 1u : 0u);
}
// D[64 x N] (+)= A^T B : rows = features [8*ga, 8*ga+64) of slab a, columns = features [8*gb, 8*gb+N) of slab b,
// contraction over the 128 rows of the tile.  `accumulate` = 0 only for the very first tile of the CTA.
template <uint32_t N>
__device__ __forceinline__ void mma_wgrad(float (&d)[N / 2], uint32_t a_s, uint32_t ga, uint32_t b_s, uint32_t gb, uint32_t accumulate) {
#pragma unroll
    for (uint32_t kb = 0; kb < ROWS / 16; ++kb)
        mma<N, 1, 1>(d, slab_desc_mnmajor(a_s, ROWS, ga, kb), slab_desc_mnmajor(b_s, ROWS, gb, kb), kb > 0 ? 1u : accumulate);
}
// One layer over a 128-row tile, one row block at a time: issue(d, m) queues the wgmmas of row block m, epi(d, m) consumes them.
// Any wgmma the warpgroup queued before (weight gradients) completes with the first block.
template <uint32_t N, class Issue, class Epi>
__device__ __forceinline__ void layer(Issue issue, Epi epi) {
#pragma unroll
    for (uint32_t m = 0; m < 2; ++m) {
        float d[N / 2];
#pragma unroll
        for (uint32_t i = 0; i < N / 2; ++i) d[i] = 0.f;
        wgmma_fence();
        issue(d, m);
        wgmma_commit();
        wgmma_wait<0>();
        epi(d, m);
    }
}

// ---- epilogue helpers (fragment layout, see wgmma.cuh; tw = thread of the warpgroup) ------------------------------
__device__ __forceinline__ uint32_t frag_row(uint32_t tw) { return 16u * (tw >> 5) + ((tw & 31u) >> 2); }
// zero the entries of packed half2 `grad` where the matching `act` half is <= 0 (ReLU')
__device__ __forceinline__ uint32_t relu_mask2(uint32_t grad, uint32_t act) {
    const __half2 a = *reinterpret_cast<const __half2*>(&act);
    const __half2 z = __float2half2_rn(0.f);
    const uint32_t m = __hgt2_mask(a, z);
    return grad & m;
}
// rows [64m, 64m+64) of D (N columns) -> fp16 (ReLU optional) -> slab groups [g0, g0+N/8)
template <uint32_t N, bool RELU>
__device__ __forceinline__ void frag_to_slab(const float (&d)[N / 2], uint8_t* slab, uint32_t g0, uint32_t m, uint32_t tw) {
    const uint32_t r = 64u * m + frag_row(tw), cb = (tw & 3u) * 4u;
#pragma unroll
    for (uint32_t c = 0; c < N / 8; ++c)
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
            float a = d[4 * c + 2 * h], b = d[4 * c + 2 * h + 1];
            if (RELU) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
            *reinterpret_cast<uint32_t*>(slab + (g0 + c) * GB + (r + 8 * h) * 16 + cb) = pack_half2(a, b);
        }
}
// dgrad epilogue: rows [64m, 64m+64) of D -> fp16 -> masked by ReLU'(act groups [ga, ..)) -> grad slab groups [g0, g0+N/8)
template <uint32_t N>
__device__ __forceinline__ void frag_dgrad_mask(const float (&d)[N / 2], const uint8_t* act_slab, uint32_t ga, uint8_t* grd_slab, uint32_t g0,
                                                uint32_t m, uint32_t tw) {
    const uint32_t r = 64u * m + frag_row(tw), cb = (tw & 3u) * 4u;
#pragma unroll
    for (uint32_t c = 0; c < N / 8; ++c)
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
            const uint32_t o = (r + 8 * h) * 16 + cb;
            const uint32_t a = *reinterpret_cast<const uint32_t*>(act_slab + (ga + c) * GB + o);
            *reinterpret_cast<uint32_t*>(grd_slab + (g0 + c) * GB + o) = relu_mask2(pack_half2(d[4 * c + 2 * h], d[4 * c + 2 * h + 1]), a);
        }
}
// row t of slab groups [g0, g0+8) -> one row-major 64-half row in global memory
__device__ __forceinline__ void slab_row_to_global(const uint8_t* slab, uint32_t g0, uint32_t t, __half* dst) {
#pragma unroll
    for (uint32_t g = 0; g < 8; ++g) reinterpret_cast<uint4*>(dst)[g] = *reinterpret_cast<const uint4*>(slab + (g0 + g) * GB + t * 16);
}
// weight-gradient fragment D[64 x N] -> fp32 reductions into dst[r * ld_r + c * ld_c] for r < r_valid, c < c_valid
template <uint32_t N>
__device__ __forceinline__ void frag_red_add(const float (&d)[N / 2], float* dst, uint32_t ld_r, uint32_t ld_c, uint32_t r_valid, uint32_t c_valid,
                                             uint32_t tw) {
    const uint32_t r0 = frag_row(tw), c0 = 2u * (tw & 3u);
#pragma unroll
    for (uint32_t c = 0; c < N / 8; ++c)
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
            for (uint32_t j = 0; j < 2; ++j) {
                const uint32_t r = r0 + 8 * h, col = 8 * c + c0 + j;
                if (r < r_valid && col < c_valid) red_add_f32(dst + r * ld_r + col * ld_c, d[4 * c + 2 * h + j]);
            }
}

// named barriers (bar.sync / bar.arrive) for warp-specialised kernels; id 0 is __syncthreads
// The barrier id is always emitted as an IMMEDIATE: with a register operand ptxas must reserve all 16 hardware barriers for the
// CTA, and barriers are an occupancy limiter -- two CTAs per SM need <= 8 each.
template <uint32_t ID>
__device__ __forceinline__ void bar_sync_imm(uint32_t nthreads) { asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(nthreads) : "memory"); }
template <uint32_t ID>
__device__ __forceinline__ void bar_arrive_imm(uint32_t nthreads) { asm volatile("bar.arrive %0, %1;" ::"n"(ID), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    switch (id) {
        case 1: bar_sync_imm<1>(nthreads); break;
        case 2: bar_sync_imm<2>(nthreads); break;
        case 3: bar_sync_imm<3>(nthreads); break;
        case 4: bar_sync_imm<4>(nthreads); break;
        case 5: bar_sync_imm<5>(nthreads); break;
        case 6: bar_sync_imm<6>(nthreads); break;
        case 7: bar_sync_imm<7>(nthreads); break;
        case 8: bar_sync_imm<8>(nthreads); break;
        case 9: bar_sync_imm<9>(nthreads); break;
        case 10: bar_sync_imm<10>(nthreads); break;
        case 11: bar_sync_imm<11>(nthreads); break;
        default: __trap();
    }
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
    switch (id) {
        case 1: bar_arrive_imm<1>(nthreads); break;
        case 2: bar_arrive_imm<2>(nthreads); break;
        case 3: bar_arrive_imm<3>(nthreads); break;
        case 4: bar_arrive_imm<4>(nthreads); break;
        case 5: bar_arrive_imm<5>(nthreads); break;
        case 6: bar_arrive_imm<6>(nthreads); break;
        case 7: bar_arrive_imm<7>(nthreads); break;
        case 8: bar_arrive_imm<8>(nthreads); break;
        case 9: bar_arrive_imm<9>(nthreads); break;
        case 10: bar_arrive_imm<10>(nthreads); break;
        case 11: bar_arrive_imm<11>(nthreads); break;
        default: __trap();
    }
}

// weight-gradient fragment D[64 x N] -> plain stores dst[r * ld_r + c * ld_c] for all 64 rows and N columns, 0 for columns >= c_valid
template <uint32_t N>
__device__ __forceinline__ void frag_store(const float (&d)[N / 2], float* dst, uint32_t ld_r, uint32_t ld_c, uint32_t c_valid, uint32_t tw) {
    const uint32_t r0 = frag_row(tw), c0 = 2u * (tw & 3u);
#pragma unroll
    for (uint32_t c = 0; c < N / 8; ++c)
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
            for (uint32_t j = 0; j < 2; ++j) {
                const uint32_t r = r0 + 8 * h, col = 8 * c + c0 + j;
                dst[r * ld_r + col * ld_c] = col < c_valid ? d[4 * c + 2 * h + j] : 0.f;
            }
}

// generic-proxy stores to operand slabs -> visible to the wgmmas of every thread that passes the barrier (0 = __syncthreads)
__device__ __forceinline__ void operands_ready(uint32_t bar_id, uint32_t nthreads) {
    fence_proxy_async_smem();
    if (bar_id == 0) __syncthreads(); else named_bar_sync(bar_id, nthreads);
}

}  // namespace mlp
