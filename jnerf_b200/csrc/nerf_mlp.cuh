// The forward half of the vanilla NeRF network kernels (nerf_mlp.cu): parameter and saved-activation layouts, the weight stream, and
// the forward kernel with its encode stage as a policy, shared by nerf_mlp.cu (FreqEnc), nerf_lattice.cu (LatticeEnc) and mip_mlp.cu
// (MipEnc), and the backward bodies.
// The encoder width is a compile-time parameter EG (8-column groups of kernel layer 0's input): 8 for NeRF and Mip-NeRF at 8 IPE
// degrees, 12 for the 96 columns of 16 degrees (mip_mlp_wide.cu).  DESIGN.md sections 10-11.
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

__host__ __device__ constexpr uint32_t in_pad(uint32_t l, uint32_t eg = 8) {
    return l == 0 ? 8 * eg : l == 5 ? 256 + 8 * eg : l == 9 ? 288 : l == 10 ? 128 : 256;
}
__host__ __device__ constexpr uint32_t out_pad(uint32_t l) { return l == 8 ? 272 : l == 9 ? 128 : l == 10 ? 16 : 256; }
__host__ __device__ constexpr uint32_t w_off(uint32_t l, uint32_t eg = 8) {
    uint32_t o = 0;
    for (uint32_t i = 0; i < l; ++i) o += out_pad(i) * (in_pad(i, eg) + 1);
    return o;
}
__host__ __device__ constexpr uint32_t b_off(uint32_t l, uint32_t eg = 8) { return w_off(l, eg) + out_pad(l) * in_pad(l, eg); }
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

// The same quantities at EG encoder groups.  The saved block puts the encoding first, so every other group base moves by EG - 8.  Past
// 8 groups the forward streams layer 5 as two K-chunks per 64 output rows (the encoding, then h4) accumulating into the same registers:
// its unsplit 64 x (256 + 8 EG) chunk would not fit beside the slabs.  The largest chunk is then views_linears.0 (64 x 288).
template <uint32_t EG>
struct Layout {
    static constexpr bool SPLIT5 = EG != 8;
    static constexpr uint32_t S_H = EG, S_F = S_H + 256, S_DIR = S_F + 32, S_V = S_DIR + 4, S_GROUPS = S_V + 16;
    static constexpr uint32_t N_PARAMS = w_off(NL, EG);
    static constexpr uint32_t FWD_CHUNKS = SPLIT5 ? 44 : 40, DENSITY_CHUNKS = FWD_CHUNKS - 7;
    static constexpr uint32_t FWD_WBUF = SPLIT5 ? 64 * 288 * 2 : 64 * in_pad(5, EG) * 2;
    static constexpr uint32_t FWD_SMEM = (EG + 32 + 32) * GB + 2 * FWD_WBUF;
    static_assert(FWD_SMEM <= 232448, "shared memory");
};
static_assert(Layout<8>::S_GROUPS == S_GROUPS && Layout<8>::S_F == S_F && Layout<8>::S_V == S_V && Layout<8>::N_PARAMS == N_PARAMS &&
              Layout<8>::FWD_SMEM == FWD_SMEM && Layout<8>::FWD_CHUNKS == FWD_CHUNKS, "layout at 8 groups");
static_assert(Layout<12>::N_PARAMS == 618912 && Layout<12>::S_GROUPS == 320 && Layout<12>::S_V == 304 && Layout<12>::FWD_SMEM == 229376,
              "layout at 12 groups");

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
// forward chunk k: 64 (or 16) output rows of one layer, all its inputs (past 8 groups layer 5 as two K-chunks, chunks 20..27)
template <uint32_t EG = 8>
__device__ __forceinline__ Chunk fwd_chunk(const __half* P, uint32_t k) {
    if constexpr (EG != 8) {
        if (k >= 20 && k < 28) {
            const uint32_t i = k - 20, c0 = (i & 1) ? 8 * EG : 0, nc = (i & 1) ? 256 : 8 * EG;
            return {P + w_off(5, EG) + 64 * (i >> 1) * in_pad(5, EG) + c0, 64, nc / 8, in_pad(5, EG)};
        }
        if (k >= 28) k -= 4;
    }
    uint32_t l, r0, nr = 64;
    if (k < 32) { l = k >> 2; r0 = 64 * (k & 3); }
    else if (k == 32) { l = 8; r0 = 0; nr = 16; }                 // alpha_linear
    else if (k < 37) { l = 8; r0 = 16 + 64 * (k - 33); }          // feature_linear
    else if (k < 39) { l = 9; r0 = 64 * (k - 37); }
    else { l = 10; r0 = 0; nr = 16; }
    return {P + w_off(l, EG) + r0 * in_pad(l, EG), nr, in_pad(l, EG) / 8, in_pad(l, EG)};
}
// dgrad chunk k: 64 input columns of one layer, all its outputs (layers 10, 9, ..., 1; layer 5 from column 8 EG: no encoder gradient)
template <uint32_t EG = 8>
__device__ __forceinline__ Chunk bwd_chunk(const __half* P, uint32_t k) {
    uint32_t l, c0;
    if (k < 2) { l = 10; c0 = 64 * k; }
    else { const uint32_t i = k - 2; l = 9 - i / 4; c0 = (l == 5 ? 8 * EG : 0) + 64 * (i & 3); }
    return {P + w_off(l, EG) + c0, out_pad(l), 8, in_pad(l, EG)};
}

// Double-buffered weight stream.  begin(): chunk k has landed and every thread is through chunk k-1 (so its buffer and the
// activations it wrote are free / visible); the load of chunk k+1 starts; returns chunk k's buffer.
template <uint32_t EG>
struct Pipe {
    uint8_t* buf[2];
    uint32_t k, n;
    const __half* P;
    bool bwd;
    __device__ __forceinline__ uint32_t begin(uint32_t tid) {
        cp_async_wait_all();
        fence_proxy_async_smem();
        __syncthreads();
        if (k + 1 < n) stage(buf[(k + 1) & 1], bwd ? bwd_chunk<EG>(P, k + 1) : fwd_chunk<EG>(P, k + 1), tid);
        return smem_u32(buf[k & 1]);
    }
    __device__ __forceinline__ void end() { ++k; }
};

// D[64 x N] = A[64 x K] W^T (ACC: D += A W^T), W chunk staged K-major with N rows
template <uint32_t N, uint32_t K, bool ACC = false, class ADesc>
__device__ __forceinline__ void gemm_fwd(float (&d)[N / 2], ADesc adesc, uint32_t w_s) {
    if constexpr (!ACC) {
#pragma unroll
        for (uint32_t i = 0; i < N / 2; ++i) d[i] = 0.f;
    }
    wgmma_fence();
#pragma unroll
    for (uint32_t kb = 0; kb < K / 16; ++kb) mma<N, 0, 0>(d, adesc(kb), slab_desc_kmajor(w_s, N, 0, kb), ACC || kb > 0 ? 1u : 0u);
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

// The encode stage of the forward kernel is a compile-time policy: pos() fills the EG input groups of pts_linears.0 (and of the skip
// layer), dir() the 4 view groups of views_linears.0; a policy used with DENSITY also stores the density kernel's output
// (store_density).  FreqEnc is vanilla NeRF's FrequencyEncoder(10) / (4) of row[0:3] / row[4:7] of `in` (stride floats a row);
// mip_mlp.cu adds the integrated positional encoding of Mip-NeRF, nerf_lattice.cu the positions of the mesh lattice.
struct FreqEnc {
    static constexpr uint32_t EG = 8;
    __device__ __forceinline__ void pos(uint8_t* slab, const float* in, uint32_t stride, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<10>(slab, [&](uint32_t row, uint32_t dim) { return in[(size_t)row * stride + dim]; }, row0, n, tid);
    }
    __device__ __forceinline__ void dir(uint8_t* slab, const float* in, uint32_t stride, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<4>(slab, [&](uint32_t row, uint32_t dim) { return in[(size_t)row * stride + 4 + dim]; }, row0, n, tid);
    }
    __device__ __forceinline__ void store_density(__half* out, uint32_t row, __half alpha) const { out[row] = alpha; }
};
__device__ __forceinline__ void slab_to_global(const uint8_t* slab, uint32_t groups, __half* dst, uint32_t tid) {
    for (uint32_t i = tid; i < groups * ROWS; i += THREADS) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(slab)[i];
}

// ---- forward: coordinate rows -> (n, 4) {rgb, alpha}, or positions -> alpha only (DENSITY) ---------------------------------------
template <bool DENSITY, bool SAVE, class Enc>
__global__ void __launch_bounds__(THREADS, 1)
    nerf_fwd_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const float* __restrict__ in, uint32_t in_stride, const __half* __restrict__ P,
                    __half* __restrict__ out, __half* __restrict__ saved, Enc enc) {
    constexpr uint32_t EG = Enc::EG;
    using L = Layout<EG>;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* X = smem;                      // enc_pos (EG groups), later enc_dir (4 groups)
    uint8_t* H0 = X + EG * GB;
    uint8_t* H1 = H0 + 32 * GB;
    uint8_t* W0 = H1 + 32 * GB;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t row0 = blockIdx.x * ROWS;
    if (row0 >= n) return;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u;
    __half* sv = SAVE ? saved + (size_t)blockIdx.x * L::S_GROUPS * ROWS * 8 : nullptr;
    Pipe<EG> pipe{{W0, W0 + L::FWD_WBUF}, 0, DENSITY ? L::DENSITY_CHUNKS : L::FWD_CHUNKS, P, false};
    stage(W0, fwd_chunk<EG>(P, 0), tid);
    enc.pos(X, in, in_stride, row0, n, tid);
    auto kmaj = [&](const uint8_t* s, uint32_t kb) { return slab_desc_kmajor(smem_u32(s) + m * 64 * 16, ROWS, 0, kb); };

    // pts_linears.0 .. 7 (ReLU); h_l goes to H[l & 1]; layer 5 reads concat([enc_pos, h4])
#pragma unroll 1
    for (uint32_t j = 0; j < 4; ++j) {
        const uint32_t w = pipe.begin(tid);
        if (SAVE && j == 0) slab_to_global(X, EG, sv + S_ENC * ROWS * 8, tid);
        float d[32];
        gemm_fwd<64, 8 * EG>(d, [&](uint32_t kb) { return kmaj(X, kb); }, w);
        epi_fwd<true, SAVE>(d, P + b_off(0, EG) + 64 * j, H0, 8 * j, sv, L::S_H + 8 * j, m, tw);
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
            if constexpr (L::SPLIT5) {
                if (l == 5) {
                    gemm_fwd<64, 8 * EG>(d, [&](uint32_t kb) { return kmaj(X, kb); }, w);
                    pipe.end();
                    gemm_fwd<64, 256, true>(d, [&](uint32_t kb) { return kmaj(src, kb); }, pipe.begin(tid));
                } else {
                    gemm_fwd<64, 256>(d, [&](uint32_t kb) { return kmaj(src, kb); }, w);
                }
            } else {
                if (l == 5) gemm_fwd<64, 320>(d, [&](uint32_t kb) { return kb < 4 ? kmaj(X, kb) : kmaj(src, kb - 4); }, w);
                else gemm_fwd<64, 256>(d, [&](uint32_t kb) { return kmaj(src, kb); }, w);
            }
            epi_fwd<true, SAVE>(d, P + b_off(l, EG) + 64 * j, dst, 8 * j, sv, L::S_H + 32 * l + 8 * j, m, tw);
            pipe.end();
        }
    }
    // alpha_linear on h7 (H1), no activation
    {
        const uint32_t w = pipe.begin(tid);
        float d[8];
        gemm_fwd<16, 256>(d, [&](uint32_t kb) { return kmaj(H1, kb); }, w);
        if ((tw & 3u) == 0) {
            const float b = __half2float(P[b_off(8, EG)]);
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h) {
                const uint32_t row = row0 + 64 * m + frag_row(tw) + 8 * h;
                if (row < n) {
                    const __half a = __float2half_rn(d[2 * h] + b);
                    if constexpr (DENSITY) enc.store_density(out, row, a);
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
            epi_fwd<false, SAVE>(d, P + b_off(8, EG) + 16 + 64 * j, H0, 8 * j, sv, L::S_F + 8 * j, m, tw);
            pipe.end();
        }
        enc.dir(X, in, in_stride, row0, n, tid);              // enc_pos is dead after layer 5
        // views_linears.0 on concat([f, enc_dir]), ReLU -> v in H1
#pragma unroll 1
        for (uint32_t j = 0; j < 2; ++j) {
            const uint32_t w = pipe.begin(tid);
            if (SAVE && j == 0) slab_to_global(X, 4, sv + L::S_DIR * ROWS * 8, tid);
            float d[32];
            gemm_fwd<64, 288>(d, [&](uint32_t kb) { return kb < 16 ? kmaj(H0, kb) : kmaj(X, kb - 16); }, w);
            epi_fwd<true, SAVE>(d, P + b_off(9, EG) + 64 * j, H1, 8 * j, sv, L::S_V + 8 * j, m, tw);
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
                        if (row < n && col < 3) out[(size_t)row * 4 + col] = __float2half_rn(d[2 * h + j] + __half2float(P[b_off(10, EG) + col]));
                    }
            }
            pipe.end();
        }
    }
}

// ---- backward 1: the dgrad chain of one tile, every layer's dY into the scratch ----------------------------------------------------
// (the body of a __global__ with __launch_bounds__(THREADS, 1) and BWD_SMEM bytes of dynamic shared memory)
template <uint32_t EG>
__device__ __forceinline__ void dgrad_body(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ P,
                                           const __half* __restrict__ saved, const __half* __restrict__ dout, __half* __restrict__ dys) {
    using L = Layout<EG>;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Ga = smem;                     // 32 groups
    uint8_t* Gb = Ga + 32 * GB;             // 34 groups: dY of kernel layer 8 = [dalpha, 0 x 15, df]
    uint8_t* S = Gb + 34 * GB;              // 2 groups: dY of rgb_linear = [drgb, 0 x 13]
    uint8_t* W0 = S + 2 * GB;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t row0 = blockIdx.x * ROWS;
    if (row0 >= n) return;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u;
    const __half* sv = saved + (size_t)blockIdx.x * L::S_GROUPS * ROWS * 8;
    __half* dy = dys + (size_t)blockIdx.x * D_GROUPS * ROWS * 8;
    Pipe<EG> pipe{{W0, W0 + BWD_WBUF}, 0, BWD_CHUNKS, P, true};
    stage(W0, bwd_chunk<EG>(P, 0), tid);
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
        epi_bwd<true>(d, sv, L::S_V + 8 * j, Ga, 8 * j, dy, D_9 + 8 * j, m, tw);
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
        epi_bwd<true>(d, sv, L::S_H + 32 * 7 + 8 * j, Ga, 8 * j, dy, D_H + 32 * 7 + 8 * j, m, tw);
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
            epi_bwd<true>(d, sv, L::S_H + 32 * (l - 1) + 8 * j, dst, 8 * j, dy, D_H + 32 * (l - 1) + 8 * j, m, tw);
            pipe.end();
        }
    }
}

// ---- backward 2: weight and bias gradients, dW_l = sum over rows of dY_l^T X_l, per row chunk --------------------------------------
// A job is (layer, 64 output rows, 128 input columns); warpgroup m takes input columns [64m, 64m+64) of it.  Chunk c of NCHUNK
// covers tiles [c T / NCHUNK, (c+1) T / NCHUNK) and writes its sums (plain stores, every parameter exactly once) to part[c].
constexpr uint32_t n_jobs(uint32_t eg = 8) {
    uint32_t s = 0;
    for (uint32_t l = 0; l < NL; ++l) s += (out_pad(l) + 63) / 64 * ((in_pad(l, eg) + 127) / 128);
    return s;
}
constexpr uint32_t WGRAD_JOBS = n_jobs();
__device__ __forceinline__ uint32_t dy_base(uint32_t l) { return l < 8 ? D_H + 32 * l : l == 8 ? D_8 : l == 9 ? D_9 : D_10; }
// saved group holding input column `col` of layer l
template <uint32_t EG>
__device__ __forceinline__ uint32_t x_group(uint32_t l, uint32_t col) {
    using L = Layout<EG>;
    if (l == 0) return S_ENC + col / 8;
    if (l == 5) return col < 8 * EG ? S_ENC + col / 8 : L::S_H + 32 * 4 + (col - 8 * EG) / 8;
    if (l == 9) return col < 256 ? L::S_F + col / 8 : L::S_DIR + (col - 256) / 8;
    if (l == 10) return L::S_V + col / 8;
    return L::S_H + 32 * (l - 1) + col / 8;
}

// (the body of a __global__ with __launch_bounds__(THREADS, 2), grid (n_jobs(EG), NCHUNK) and WGRAD_SMEM bytes of dynamic shared memory)
template <uint32_t EG>
__device__ __forceinline__ void wgrad_body(uint32_t n_max, const uint32_t* __restrict__ n_dev, const __half* __restrict__ saved,
                                           const __half* __restrict__ dys, float* __restrict__ part) {
    using L = Layout<EG>;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* A[2] = {smem, smem + 8 * GB};
    uint8_t* B[2] = {smem + 16 * GB, smem + 32 * GB};
    uint32_t idx = blockIdx.x, l = 0;
    for (;; ++l) {
        const uint32_t nj = (out_pad(l) + 63) / 64 * ((in_pad(l, EG) + 127) / 128);
        if (idx < nj) break;
        idx -= nj;
    }
    const uint32_t nib = (in_pad(l, EG) + 127) / 128, ob = idx / nib, ib = idx % nib;
    const uint32_t in = in_pad(l, EG), outp = out_pad(l), c = blockIdx.y;
    const uint32_t tid = threadIdx.x, m = tid >> 7, tw = tid & 127u, col_wg = 128 * ib + 64 * m;
    const uint32_t n = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t T = (n + ROWS - 1) / ROWS, t0 = (uint32_t)((uint64_t)c * T / NCHUNK), t1 = (uint32_t)((uint64_t)(c + 1) * T / NCHUNK);
    auto stage_tile = [&](uint32_t t, uint32_t b) {
        const __half* a_src = dys + ((size_t)t * D_GROUPS + dy_base(l) + 8 * ob) * ROWS * 8;
        for (uint32_t i = tid; i < 8 * ROWS; i += THREADS) cp_async16(smem_u32(A[b]) + i * 16, a_src + (size_t)i * 8);
        for (uint32_t i = tid; i < 16 * ROWS; i += THREADS) {
            const uint32_t col = 128 * ib + 8 * (i / ROWS);
            if (col < in) cp_async16(smem_u32(B[b]) + i * 16, saved + ((size_t)t * L::S_GROUPS + x_group<EG>(l, col)) * ROWS * 8 + (i % ROWS) * 8);
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
    float* dst = part + (size_t)c * L::N_PARAMS;
    if (active) {
        const uint32_t r0 = frag_row(tw), c0 = 2 * (tw & 3u);
#pragma unroll
        for (uint32_t cc = 0; cc < 8; ++cc)
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
                for (uint32_t j = 0; j < 2; ++j) {
                    const uint32_t orow = 64 * ob + r0 + 8 * h, icol = col_wg + 8 * cc + c0 + j;
                    if (orow < outp && icol < in) dst[w_off(l, EG) + orow * in + icol] = d[4 * cc + 2 * h + j];
                }
    }
    if (bias_thread && 64 * ob + tw < outp) dst[b_off(l, EG) + 64 * ob + tw] = bsum;
}

template <uint32_t EG>
__device__ __forceinline__ void wgrad_reduce_body(const float* __restrict__ part, float* __restrict__ grad) {
    constexpr uint32_t NP = Layout<EG>::N_PARAMS;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NP) return;
    float s = part[i];
#pragma unroll
    for (uint32_t c = 1; c < NCHUNK; ++c) s += part[(size_t)c * NP + i];
    grad[i] = s;
}

inline uint64_t tiles(uint32_t n) { return (n + ROWS - 1) / ROWS; }

template <bool DENSITY, bool SAVE, class Enc = FreqEnc>
int launch_fwd(cudaStream_t s, uint32_t n_max, const uint32_t* n_dev, const float* in, uint32_t stride, const void* params, void* out, void* saved,
               Enc enc = Enc{}) {
    auto k = nerf_fwd_kernel<DENSITY, SAVE, Enc>;
    constexpr uint32_t smem_bytes = Layout<Enc::EG>::FWD_SMEM;
    if (ngp_first_use((const void*)k)) NGP_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    k<<<(uint32_t)tiles(n_max), THREADS, smem_bytes, s>>>(n_max, n_dev, in, stride, (const __half*)params, (__half*)out, (__half*)saved, enc);
    NGP_LAUNCH_CHECK();
    return 0;
}
}  // namespace nerf
