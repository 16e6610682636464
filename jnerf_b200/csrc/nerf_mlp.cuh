// The forward half of the vanilla NeRF network kernels (nerf_mlp.cu): parameter and saved-activation layouts, the weight stream, and
// the forward kernel with its encode stage as a policy, shared by nerf_mlp.cu (FreqEnc) and mip_mlp.cu (MipEnc).  DESIGN.md sections 10-11.
#pragma once
#include "mlp_tc.cuh"
#include "ngp_b200.h"

namespace nerf {
using namespace wg;
using mlp::GB;
using mlp::ROWS;
using mlp::frag_row;

constexpr uint32_t THREADS = 256;
constexpr uint32_t NL = 11;

__host__ __device__ constexpr uint32_t in_pad(uint32_t l) { return l == 0 ? 64 : l == 5 ? 320 : l == 9 ? 288 : l == 10 ? 128 : 256; }
__host__ __device__ constexpr uint32_t out_pad(uint32_t l) { return l == 8 ? 272 : l == 9 ? 128 : l == 10 ? 16 : 256; }
__host__ __device__ constexpr uint32_t w_off(uint32_t l) {
    uint32_t o = 0;
    for (uint32_t i = 0; i < l; ++i) o += out_pad(i) * (in_pad(i) + 1);
    return o;
}
__host__ __device__ constexpr uint32_t b_off(uint32_t l) { return w_off(l) + out_pad(l) * in_pad(l); }
constexpr uint32_t N_PARAMS = w_off(NL);
static_assert(N_PARAMS == 602528, "parameter layout");

// Saved forward activations (the input of every layer), per 128-row tile one block in slab layout: feature group g of the block is
// [128 rows][8 halfs].  Group bases:
constexpr uint32_t S_ENC = 0, S_H = 8 /* + 32 l: h_l = ReLU output of trunk layer l */, S_F = 264, S_DIR = 296, S_V = 300, S_GROUPS = 316;
// Pre-activation gradients dY of every layer (the wgrad GEMM's other operand), same block layout:
constexpr uint32_t D_H = 0 /* + 32 l */, D_8 = 256 /* 40 groups: alpha, 0, df, 0 */, D_9 = 296, D_10 = 312 /* 8 groups: drgb, 0 */, D_GROUPS = 320;
// weight-gradient partial sums: a fixed number of row chunks, summed in chunk order (deterministic, no float atomics)
constexpr uint32_t NCHUNK = 8;

constexpr uint32_t FWD_CHUNKS = 40, DENSITY_CHUNKS = 33, BWD_CHUNKS = 38;
constexpr uint32_t FWD_WBUF = 64 * 320 * 2;           // largest forward chunk: 64 rows of pts_linears.5
constexpr uint32_t BWD_WBUF = 272 * 64 * 2;           // largest dgrad chunk: 64 columns of kernel layer 8
constexpr uint32_t FWD_SMEM = (8 + 32 + 32) * GB + 2 * FWD_WBUF;
constexpr uint32_t BWD_SMEM = (32 + 34 + 2) * GB + 2 * BWD_WBUF;
constexpr uint32_t WGRAD_SMEM = 2 * (8 + 16) * GB;
static_assert(FWD_SMEM <= 232448 && BWD_SMEM <= 232448, "shared memory");

// ---- cp.async -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// A weight chunk: rows [0, nrows) x groups [0, ngroups) of a row-major matrix with `stride` halfs per row -> smem [ngroups][nrows][8].
// Eight consecutive threads copy one group of eight consecutive rows: 128 contiguous bytes in shared memory, 64-byte runs in global.
struct Chunk {
    const __half* src;
    uint32_t nrows, ngroups, stride;
};
__device__ __forceinline__ void stage(uint8_t* dst, Chunk c, uint32_t tid) {
    const uint32_t d = smem_u32(dst), n = c.nrows * c.ngroups;
    for (uint32_t i = tid; i < n; i += THREADS) {
        const uint32_t rest = i >> 3, g = rest % c.ngroups, r = (rest / c.ngroups) * 8 + (i & 7);
        cp_async16(d + (g * c.nrows + r) * 16, c.src + (size_t)r * c.stride + g * 8);
    }
    cp_async_commit();
}
// forward chunk k: 64 (or 16) output rows of one layer, all its inputs
__device__ __forceinline__ Chunk fwd_chunk(const __half* P, uint32_t k) {
    uint32_t l, r0, nr = 64;
    if (k < 32) { l = k >> 2; r0 = 64 * (k & 3); }
    else if (k == 32) { l = 8; r0 = 0; nr = 16; }                 // alpha_linear
    else if (k < 37) { l = 8; r0 = 16 + 64 * (k - 33); }          // feature_linear
    else if (k < 39) { l = 9; r0 = 64 * (k - 37); }
    else { l = 10; r0 = 0; nr = 16; }
    return {P + w_off(l) + r0 * in_pad(l), nr, in_pad(l) / 8, in_pad(l)};
}
// dgrad chunk k: 64 input columns of one layer, all its outputs (layers 10, 9, ..., 1; layer 5 from column 64: no encoder gradient)
__device__ __forceinline__ Chunk bwd_chunk(const __half* P, uint32_t k) {
    uint32_t l, c0;
    if (k < 2) { l = 10; c0 = 64 * k; }
    else { const uint32_t i = k - 2; l = 9 - i / 4; c0 = (l == 5 ? 64 : 0) + 64 * (i & 3); }
    return {P + w_off(l) + c0, out_pad(l), 8, in_pad(l)};
}

// Double-buffered weight stream.  begin(): chunk k has landed and every thread is through chunk k-1 (so its buffer and the
// activations it wrote are free / visible); the load of chunk k+1 starts; returns chunk k's buffer.
struct Pipe {
    uint8_t* buf[2];
    uint32_t k, n;
    const __half* P;
    bool bwd;
    __device__ __forceinline__ uint32_t begin(uint32_t tid) {
        cp_async_wait_all();
        fence_proxy_async_smem();
        __syncthreads();
        if (k + 1 < n) stage(buf[(k + 1) & 1], bwd ? bwd_chunk(P, k + 1) : fwd_chunk(P, k + 1), tid);
        return smem_u32(buf[k & 1]);
    }
    __device__ __forceinline__ void end() { ++k; }
};

// D[64 x N] = A[64 x K] W^T, W chunk staged K-major with N rows
template <uint32_t N, uint32_t K, class ADesc>
__device__ __forceinline__ void gemm_fwd(float (&d)[N / 2], ADesc adesc, uint32_t w_s) {
#pragma unroll
    for (uint32_t i = 0; i < N / 2; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (uint32_t kb = 0; kb < K / 16; ++kb) mma<N, 0, 0>(d, adesc(kb), slab_desc_kmajor(w_s, N, 0, kb), kb > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
}
// D[64 x N] = dY[64 x K] W[K x N], W chunk staged with K rows, read MN-major
template <uint32_t N, uint32_t K, class ADesc>
__device__ __forceinline__ void gemm_bwd(float (&d)[N / 2], ADesc adesc, uint32_t w_s) {
#pragma unroll
    for (uint32_t i = 0; i < N / 2; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (uint32_t kb = 0; kb < K / 16; ++kb) mma<N, 0, 1>(d, adesc(kb), slab_desc_mnmajor(w_s, K, 0, kb), kb > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
}

// bias in fp32 on the accumulator, optional ReLU, one rounding to fp16 -> slab groups [og, og+8) (+ the saved block, groups [sg, ..))
template <bool RELU, bool SAVE>
__device__ __forceinline__ void epi_fwd(const float (&d)[32], const __half* bias, uint8_t* slab, uint32_t og, __half* save, uint32_t sg,
                                        uint32_t m, uint32_t tw) {
    const uint32_t r = 64u * m + frag_row(tw), cb = (tw & 3u) * 4u;
#pragma unroll
    for (uint32_t c = 0; c < 8; ++c) {
        const float2 b = __half22float2(__ldg(reinterpret_cast<const __half2*>(bias + 8 * c + 2 * (tw & 3u))));
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
            float a = d[4 * c + 2 * h] + b.x, e = d[4 * c + 2 * h + 1] + b.y;
            if (RELU) { a = fmaxf(a, 0.f); e = fmaxf(e, 0.f); }
            const uint32_t u = pack_half2(a, e), o = (r + 8 * h) * 16 + cb;
            *reinterpret_cast<uint32_t*>(slab + (og + c) * GB + o) = u;
            if (SAVE) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(save) + (sg + c) * GB + o) = u;
        }
    }
}
// dX -> fp16 -> (masked by ReLU' of the saved activation groups [mg, ..)) -> slab groups [og, ..) and the dY block groups [dg, ..)
template <bool MASK>
__device__ __forceinline__ void epi_bwd(const float (&d)[32], const __half* act, uint32_t mg, uint8_t* slab, uint32_t og, __half* dy, uint32_t dg,
                                        uint32_t m, uint32_t tw) {
    const uint32_t r = 64u * m + frag_row(tw), cb = (tw & 3u) * 4u;
#pragma unroll
    for (uint32_t c = 0; c < 8; ++c)
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
            const uint32_t o = (r + 8 * h) * 16 + cb;
            uint32_t u = pack_half2(d[4 * c + 2 * h], d[4 * c + 2 * h + 1]);
            if (MASK) u = mlp::relu_mask2(u, __ldg(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(act) + (mg + c) * GB + o)));
            *reinterpret_cast<uint32_t*>(slab + (og + c) * GB + o) = u;
            *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(dy) + (dg + c) * GB + o) = u;
        }
}

// enc(x) = [x, sin(x 2^0), cos(x 2^0), ..., sin(x 2^(L-1)), cos(x 2^(L-1))], 3 wide each, in fp32 with the full-range sincosf
// (arguments reach 512 rad), rounded once to fp16; columns past 3 + 6L are zero.  Rows at or past n encode x = 0.  x(row, dim) reads
// coordinate dim of tile row `row` (absolute row index).
template <uint32_t L, class X>
__device__ __forceinline__ void encode_rows(uint8_t* slab, X xat, uint32_t row0, uint32_t n, uint32_t tid) {
    constexpr uint32_t W = 3 + 6 * L, WP = (W + 7) / 8 * 8;
    for (uint32_t t = tid; t < ROWS * 3; t += THREADS) {
        const uint32_t r = t / 3, dim = t % 3;
        const float x = row0 + r < n ? xat(row0 + r, dim) : 0.f;
        auto put = [&](uint32_t f, float v) { *reinterpret_cast<__half*>(slab + (f / 8) * GB + r * 16 + (f % 8) * 2) = __float2half_rn(v); };
        put(dim, x);
#pragma unroll
        for (uint32_t k = 0; k < L; ++k) {
            float s, c;
            sincosf(x * (float)(1u << k), &s, &c);
            put(3 + 6 * k + dim, s);
            put(6 + 6 * k + dim, c);
        }
        if (dim == 0)
            for (uint32_t f = W; f < WP; ++f) put(f, 0.f);
    }
}

// The encode stage of the forward kernel is a compile-time policy: pos() fills the 8 input groups of pts_linears.0 (and of the skip
// layer), dir() the 4 view groups of views_linears.0.  FreqEnc is vanilla NeRF's FrequencyEncoder(10) / (4) of row[0:3] / row[4:7] of
// `in` (stride floats a row); mip_mlp.cu adds the integrated positional encoding of Mip-NeRF.
struct FreqEnc {
    __device__ __forceinline__ void pos(uint8_t* slab, const float* in, uint32_t stride, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<10>(slab, [&](uint32_t row, uint32_t dim) { return in[(size_t)row * stride + dim]; }, row0, n, tid);
    }
    __device__ __forceinline__ void dir(uint8_t* slab, const float* in, uint32_t stride, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<4>(slab, [&](uint32_t row, uint32_t dim) { return in[(size_t)row * stride + 4 + dim]; }, row0, n, tid);
    }
};
__device__ __forceinline__ void slab_to_global(const uint8_t* slab, uint32_t groups, __half* dst, uint32_t tid) {
    for (uint32_t i = tid; i < groups * ROWS; i += THREADS) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(slab)[i];
}

// ---- forward: coordinate rows -> (n, 4) {rgb, alpha}, or positions -> alpha only (DENSITY) ---------------------------------------
template <bool DENSITY, bool SAVE, class Enc>
__global__ void __launch_bounds__(THREADS, 1)
    nerf_fwd_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const float* __restrict__ in, uint32_t in_stride, const __half* __restrict__ P,
                    __half* __restrict__ out, __half* __restrict__ saved, Enc enc) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* X = smem;                      // enc_pos (8 groups), later enc_dir (4 groups)
    uint8_t* H0 = X + 8 * GB;
    uint8_t* H1 = H0 + 32 * GB;
    uint8_t* W0 = H1 + 32 * GB;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t row0 = blockIdx.x * ROWS;
    if (row0 >= n) return;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u;
    __half* sv = SAVE ? saved + (size_t)blockIdx.x * S_GROUPS * ROWS * 8 : nullptr;
    Pipe pipe{{W0, W0 + FWD_WBUF}, 0, DENSITY ? DENSITY_CHUNKS : FWD_CHUNKS, P, false};
    stage(W0, fwd_chunk(P, 0), tid);
    enc.pos(X, in, in_stride, row0, n, tid);
    auto kmaj = [&](const uint8_t* s, uint32_t kb) { return slab_desc_kmajor(smem_u32(s) + m * 64 * 16, ROWS, 0, kb); };

    // pts_linears.0 .. 7 (ReLU); h_l goes to H[l & 1]; layer 5 reads concat([enc_pos, h4])
#pragma unroll 1
    for (uint32_t j = 0; j < 4; ++j) {
        const uint32_t w = pipe.begin(tid);
        if (SAVE && j == 0) slab_to_global(X, 8, sv + S_ENC * ROWS * 8, tid);
        float d[32];
        gemm_fwd<64, 64>(d, [&](uint32_t kb) { return kmaj(X, kb); }, w);
        epi_fwd<true, SAVE>(d, P + b_off(0) + 64 * j, H0, 8 * j, sv, S_H + 8 * j, m, tw);
        pipe.end();
    }
#pragma unroll 1
    for (uint32_t l = 1; l < 8; ++l) {
        uint8_t* src = (l & 1) ? H0 : H1;
        uint8_t* dst = (l & 1) ? H1 : H0;
#pragma unroll 1
        for (uint32_t j = 0; j < 4; ++j) {
            const uint32_t w = pipe.begin(tid);
            float d[32];
            if (l == 5) gemm_fwd<64, 320>(d, [&](uint32_t kb) { return kb < 4 ? kmaj(X, kb) : kmaj(src, kb - 4); }, w);
            else gemm_fwd<64, 256>(d, [&](uint32_t kb) { return kmaj(src, kb); }, w);
            epi_fwd<true, SAVE>(d, P + b_off(l) + 64 * j, dst, 8 * j, sv, S_H + 32 * l + 8 * j, m, tw);
            pipe.end();
        }
    }
    // alpha_linear on h7 (H1), no activation
    {
        const uint32_t w = pipe.begin(tid);
        float d[8];
        gemm_fwd<16, 256>(d, [&](uint32_t kb) { return kmaj(H1, kb); }, w);
        if ((tw & 3u) == 0) {
            const float b = __half2float(P[b_off(8)]);
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h) {
                const uint32_t row = row0 + 64 * m + frag_row(tw) + 8 * h;
                if (row < n) {
                    const __half a = __float2half_rn(d[2 * h] + b);
                    if (DENSITY) out[row] = a;
                    else out[(size_t)row * 4 + 3] = a;
                }
            }
        }
        pipe.end();
    }
    if constexpr (!DENSITY) {
        // feature_linear on h7, no activation -> f in H0
#pragma unroll 1
        for (uint32_t j = 0; j < 4; ++j) {
            const uint32_t w = pipe.begin(tid);
            float d[32];
            gemm_fwd<64, 256>(d, [&](uint32_t kb) { return kmaj(H1, kb); }, w);
            epi_fwd<false, SAVE>(d, P + b_off(8) + 16 + 64 * j, H0, 8 * j, sv, S_F + 8 * j, m, tw);
            pipe.end();
        }
        enc.dir(X, in, in_stride, row0, n, tid);              // enc_pos is dead after layer 5
        // views_linears.0 on concat([f, enc_dir]), ReLU -> v in H1
#pragma unroll 1
        for (uint32_t j = 0; j < 2; ++j) {
            const uint32_t w = pipe.begin(tid);
            if (SAVE && j == 0) slab_to_global(X, 4, sv + S_DIR * ROWS * 8, tid);
            float d[32];
            gemm_fwd<64, 288>(d, [&](uint32_t kb) { return kb < 16 ? kmaj(H0, kb) : kmaj(X, kb - 16); }, w);
            epi_fwd<true, SAVE>(d, P + b_off(9) + 64 * j, H1, 8 * j, sv, S_V + 8 * j, m, tw);
            pipe.end();
        }
        // rgb_linear, no activation
        {
            const uint32_t w = pipe.begin(tid);
            float d[8];
            gemm_fwd<16, 128>(d, [&](uint32_t kb) { return kmaj(H1, kb); }, w);
            if ((tw & 3u) < 2) {
#pragma unroll
                for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
                    for (uint32_t j = 0; j < 2; ++j) {
                        const uint32_t row = row0 + 64 * m + frag_row(tw) + 8 * h, col = 2 * (tw & 3u) + j;
                        if (row < n && col < 3) out[(size_t)row * 4 + col] = __float2half_rn(d[2 * h + j] + __half2float(P[b_off(10) + col]));
                    }
            }
            pipe.end();
        }
    }
}

inline uint64_t tiles(uint32_t n) { return (n + ROWS - 1) / ROWS; }

template <bool DENSITY, bool SAVE, class Enc = FreqEnc>
int launch_fwd(cudaStream_t s, uint32_t n_max, const uint32_t* n_dev, const float* in, uint32_t stride, const void* params, void* out, void* saved,
               Enc enc = Enc{}) {
    auto k = nerf_fwd_kernel<DENSITY, SAVE, Enc>;
    if (ngp_first_use((const void*)k)) NGP_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM));
    k<<<(uint32_t)tiles(n_max), THREADS, FWD_SMEM, s>>>(n_max, n_dev, in, stride, (const __half*)params, (__half*)out, (__half*)saved, enc);
    NGP_LAUNCH_CHECK();
    return 0;
}
}  // namespace nerf
