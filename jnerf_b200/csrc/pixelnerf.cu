// pixelNeRF (contrib/pixelnerf: Network.py, Render.py, Dataset.py:74-94) on sm_90a.  DESIGN.md section 13.
//
// Every 512-wide layer is one launch of pn_gemm_kernel: a 128x128 CTA tile, two consumer warpgroups of m64n128k16 wgmma, fp32
// accumulators, K streamed in 64-column steps through a 3-stage cp.async ring of operand slabs (wgmma.cuh's un-swizzled layout).  What
// differs between layers is where the A / B tiles come from and what the epilogue does:
//   - the W_img layers read their A operand (forward) or B operand (wgrad) from the gather: the sample's four bilinear taps into the
//     channel-last fp16 feature maps, blended in fp32 and rounded once to fp16 in shared memory.  The (n_ref, R S, 512) features never exist
//     in HBM;
//   - forward epilogues: bias + ReLU, then the residual add (the stem output broadcast over the references in block 0 of f1);
//   - dgrad epilogues: the residual gradient added in fp32, the ReLU masks of the saved activations;
//   - wgrad: blockIdx.z is one of a fixed number of row chunks, written as fp32 partials and summed in chunk order (pn_reduce_kernel).
// Rows are reference-major: reference row q = k * Ms + j for reference k and sample row j = ray * S + sample.
#include <cuda_fp16.h>
#include <stdint.h>

#include "ngp_b200.h"
#include "ngp_common.cuh"
#include "wgmma.cuh"

namespace pn {

constexpr uint32_t WIDTH = 512, ENC_PAD = 64, ENC_COLS = 42, HEAD_PAD = 8;
constexpr uint32_t N_F1 = 3, N_F2 = 2;
constexpr uint32_t LIN = WIDTH * WIDTH + WIDTH;                                   // one 512x512 Linear with its bias
// flat fp16 parameters: mlp.0 (512 x 64, columns 42..63 zero), f1.i (img_mlp.0, mlp.0, mlp.2), f2.i (mlp.0, mlp.2), final_layer (4 x 512)
constexpr uint32_t P_STEM = 0, P_F1 = WIDTH * ENC_PAD + WIDTH, P_F2 = P_F1 + N_F1 * 3 * LIN, P_HEAD = P_F2 + N_F2 * 2 * LIN;
constexpr uint32_t N_PARAMS = P_HEAD + 4 * WIDTH + 4;
constexpr uint32_t BM = 128, BN = 128, BK = 64, STAGES = 3, THREADS = 256;
constexpr uint32_t SLAB = BM * BK * 2;                                           // one operand tile: 16 KB
constexpr uint32_t GEMM_SMEM = STAGES * 2 * SLAB;                                // 96 KB: two CTAs an SM
constexpr uint32_t WG_CHUNKS = 16;                                               // wgrad row chunks
constexpr uint32_t CS_CHUNKS = 128;                                              // bias-gradient row chunks

enum { EPI_FWD = 0, EPI_HEAD = 1, EPI_BWD = 2, EPI_WGRAD = 3 };

struct Gather {
    const int4* taps;        // per reference row: the four texel offsets (in halfs) of (y0,x0) (y0,x1) (y1,x0) (y1,x1)
    const float4* tapw;      // ... and their bilinear weights
    const __half* feats;     // (n_ref, fh, fw, 512) fp16
};

struct GemmArgs {
    const __half* A;         // TA = 0: (M, K) row-major; TA = 1: (K, M) row-major
    const __half* B;         // TB = 0: (N, K) row-major; TB = 1: (K, N) row-major
    uint32_t lda, ldb, M, N, K, kb_lim;   // kb_lim: rows of B that exist when TB = 1 (the rest read zero)
    int gather_a, gather_b;  // the operand comes from the gather instead of A / B
    Gather g;
    const __half* bias;
    const __half* res;       // forward: residual (out1 = res + relu(...)); backward: added gradient.  Row m reads row m % res_rows.
    uint32_t res_rows;
    float res_scale;
    __half *out0, *out1, *out2;           // NULL: not written
    const __half *mask1, *mask2;          // backward: out1 = v [mask1 > 0], out2 = v [mask2 > 0]
    uint32_t ldo;
    float* part;             // wgrad: (gridDim.z, M, N) fp32
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16u : 0u) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int TA, int TB>
__device__ __forceinline__ void mma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, "
        "%28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, "
        "%54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
          "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

// Eight channels [c0, c0 + 8) of reference row q, bilinear in fp32 over the four taps, rounded once to fp16.
__device__ __forceinline__ uint4 gather8(const Gather& g, uint32_t q, uint32_t c0) {
    const int4 t = g.taps[q];
    const float4 w = g.tapw[q];
    const int off[4] = {t.x, t.y, t.z, t.w};
    const float wt[4] = {w.x, w.y, w.z, w.w};
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(g.feats + off[k] + c0));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            acc[2 * e] = fmaf(wt[k], f.x, acc[2 * e]);
            acc[2 * e + 1] = fmaf(wt[k], f.y, acc[2 * e + 1]);
        }
    }
    uint4 o;
    o.x = wg::pack_half2(acc[0], acc[1]);
    o.y = wg::pack_half2(acc[2], acc[3]);
    o.z = wg::pack_half2(acc[4], acc[5]);
    o.w = wg::pack_half2(acc[6], acc[7]);
    return o;
}

// One operand tile into a slab.  T = 0: 128 slab rows = rows [mn0, +128) of a row-major (MN, K) matrix, 8 groups = columns [k0, +64).
// T = 1: 64 slab rows = rows [k0, +64) of a row-major (K, MN) matrix, 16 groups = columns [mn0, +128).  Out-of-range chunks read zero.
// Each warp covers 8 rows x 4 groups: a quarter-warp stores 128 contiguous bytes, a row's 4 groups are 64 contiguous bytes in HBM.
template <int T>
__device__ __forceinline__ void load_tile(uint32_t slab, const __half* src, uint32_t ld, uint32_t mn0, uint32_t k0, uint32_t mn_lim,
                                          uint32_t k_lim, const Gather* g, uint32_t tid) {
    constexpr uint32_t R = T == 0 ? BM : BK, RB = R / 8;
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t c = tid + THREADS * i, lane = c & 31, w = c >> 5;
        const uint32_t r = (w % RB) * 8 + (lane & 7), gi = (w / RB) * 4 + (lane >> 3);
        const uint32_t srow = T == 0 ? mn0 + r : k0 + r, scol = T == 0 ? k0 + 8 * gi : mn0 + 8 * gi;
        const uint32_t row_lim = T == 0 ? mn_lim : k_lim, col_lim = T == 0 ? k_lim : mn_lim;
        const bool ok = srow < row_lim && scol < col_lim;
        const uint32_t dst = slab + gi * (R * 16) + r * 16;
        if (g) {
            uint4 v = make_uint4(0, 0, 0, 0);
            if (ok) v = gather8(*g, srow, scol);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        } else {
            cp_async16(dst, ok ? src + (size_t)srow * ld + scol : src, ok);
        }
    }
}

template <int EPI>
__global__ void __launch_bounds__(THREADS, 2) pn_gemm_kernel(const GemmArgs p) {
    constexpr int TA = EPI == EPI_WGRAD ? 1 : 0, TB = EPI >= EPI_BWD ? 1 : 0;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t tid = threadIdx.x, wgi = tid / 128, t = tid % 128;
    const uint32_t n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
    const uint32_t steps = (p.K + BK - 1) / BK;
    const uint32_t ks0 = (uint32_t)((uint64_t)steps * blockIdx.z / gridDim.z), ks1 = (uint32_t)((uint64_t)steps * (blockIdx.z + 1) / gridDim.z);
    const uint32_t nk = ks1 - ks0;
    const uint32_t base = wg::smem_u32(smem);
    const Gather* ga = p.gather_a ? &p.g : nullptr;
    const Gather* gb = p.gather_b ? &p.g : nullptr;
    const uint32_t kb_lim = TB == 1 ? p.kb_lim : p.K;

    auto load_stage = [&](uint32_t slot, uint32_t ks) {
        const uint32_t a_s = base + slot * 2 * SLAB, b_s = a_s + SLAB, k0 = ks * BK;
        load_tile<TA>(a_s, p.A, p.lda, m0, k0, p.M, p.K, ga, tid);
        load_tile<TB>(b_s, p.B, p.ldb, n0, k0, p.N, kb_lim, gb, tid);
    };

    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;

#pragma unroll
    for (uint32_t s = 0; s < STAGES - 1; ++s) {
        if (s < nk) load_stage(s, ks0 + s);
        cp_async_commit();
    }
#pragma unroll 1
    for (uint32_t it = 0; it < nk; ++it) {
        cp_async_wait<STAGES - 2>();
        wg::fence_proxy_async_smem();
        __syncthreads();
        const uint32_t slot = it % STAGES, a_s = base + slot * 2 * SLAB, b_s = a_s + SLAB;
        wg::wgmma_fence();
#pragma unroll
        for (uint32_t kb = 0; kb < BK / 16; ++kb) {
            const uint64_t da = TA == 0 ? wg::slab_desc_kmajor(a_s + wgi * 64 * 16, BM, 0, kb) : wg::slab_desc_mnmajor(a_s, BK, 8 * wgi, kb);
            const uint64_t db = TB == 0 ? wg::slab_desc_kmajor(b_s, BN, 0, kb) : wg::slab_desc_mnmajor(b_s, BK, 0, kb);
            mma_n128<TA, TB>(d, da, db, 1u);
        }
        wg::wgmma_commit();
        // the slot refilled here was read by iteration it - 1, whose wgmmas every thread waited for before the barrier above
        if (it + STAGES - 1 < nk) load_stage((it + STAGES - 1) % STAGES, ks0 + it + STAGES - 1);
        cp_async_commit();
        wg::wgmma_wait<0>();
    }
    cp_async_wait<0>();

    // thread t of warpgroup wgi holds d[4c + 2h + j] = D[64 wgi + 16 (t / 32) + (t % 32) / 4 + 8 h][8 c + 2 (t % 4) + j]
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
        const uint32_t m = m0 + 64 * wgi + 16 * (t / 32) + (t % 32) / 4 + 8 * h;
        if (m >= p.M) continue;
#pragma unroll
        for (uint32_t c = 0; c < 16; ++c) {
            const uint32_t n = n0 + 8 * c + 2 * (t % 4);
            if (n >= p.N) continue;
            float v0 = d[4 * c + 2 * h], v1 = d[4 * c + 2 * h + 1];
            if constexpr (EPI == EPI_WGRAD) {
                *reinterpret_cast<float2*>(p.part + ((size_t)blockIdx.z * p.M + m) * p.N + n) = make_float2(v0, v1);
            } else if constexpr (EPI == EPI_HEAD) {
                // final_layer: sigma = relu(o0), c = sigmoid(o1:4); N = 4, raw rows of 4 halfs
                v0 += __half2float(p.bias[n]);
                v1 += __half2float(p.bias[n + 1]);
                v0 = n == 0 ? fmaxf(v0, 0.f) : 1.f / (1.f + expf(-v0));
                v1 = 1.f / (1.f + expf(-v1));
                *reinterpret_cast<__half2*>(p.out0 + (size_t)m * 4 + n) = __floats2half2_rn(v0, v1);
            } else if constexpr (EPI == EPI_FWD) {
                const float2 b = __half22float2(*reinterpret_cast<const __half2*>(p.bias + n));
                const __half2 y = __floats2half2_rn(fmaxf(v0 + b.x, 0.f), fmaxf(v1 + b.y, 0.f));
                const size_t o = (size_t)m * p.ldo + n;
                if (p.out0) *reinterpret_cast<__half2*>(p.out0 + o) = y;
                if (p.res) {
                    const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.res + (size_t)(m % p.res_rows) * p.ldo + n));
                    const float2 yf = __half22float2(y);
                    *reinterpret_cast<__half2*>(p.out1 + o) = __floats2half2_rn(r.x + yf.x, r.y + yf.y);
                }
            } else {  // EPI_BWD
                if (p.res) {
                    const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.res + (size_t)(m % p.res_rows) * p.ldo + n));
                    v0 = fmaf(p.res_scale, r.x, v0);
                    v1 = fmaf(p.res_scale, r.y, v1);
                }
                const __half2 y = __floats2half2_rn(v0, v1), z = __float2half2_rn(0.f);
                const size_t o = (size_t)m * p.ldo + n;
                if (p.out0) *reinterpret_cast<__half2*>(p.out0 + o) = y;
                if (p.out1) {
                    const __half2 k = *reinterpret_cast<const __half2*>(p.mask1 + o);
                    *reinterpret_cast<__half2*>(p.out1 + o) = __halves2half2(__hgt(__low2half(k), __float2half(0.f)) ? __low2half(y) : __low2half(z),
                                                                             __hgt(__high2half(k), __float2half(0.f)) ? __high2half(y) : __high2half(z));
                }
                if (p.out2) {
                    const __half2 k = *reinterpret_cast<const __half2*>(p.mask2 + o);
                    *reinterpret_cast<__half2*>(p.out2 + o) = __halves2half2(__hgt(__low2half(k), __float2half(0.f)) ? __low2half(y) : __low2half(z),
                                                                             __hgt(__high2half(k), __float2half(0.f)) ? __high2half(y) : __high2half(z));
                }
            }
        }
    }
}

// ---- the small kernels -------------------------------------------------------------------------------------------------------------------

// Dataset.py:86-94 for reference row q: project the sample into reference k, grid_sample(align_corners=True, padding_mode="border")'s
// four taps.  cams (n_ref, 12): R_t row-major, then the camera position.  A non-finite coordinate (p.z = 0) clamps to the border, as
// torch's CUDA grid_sample does (fmaxf(NaN, 0) = 0).
__global__ void pn_taps_kernel(uint32_t Ms, uint32_t S, uint32_t n_ref, const float* __restrict__ rays, const float* __restrict__ z,
                               const float* __restrict__ cams, uint32_t fh, uint32_t fw, float scale, int pixel_aligned, int4* __restrict__ taps,
                               float4* __restrict__ tapw) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Ms * n_ref) return;
    const uint32_t k = q / Ms, j = q % Ms, ray = j / S, s = j % S;
    const float* r = rays + (size_t)ray * 6;
    const float zz = z[s];
    const float x[3] = {r[0] + r[3] * zz, r[1] + r[4] * zz, r[2] + r[5] * zz};
    const float* c = cams + k * 12;
    const float e[3] = {x[0] - c[9], x[1] - c[10], x[2] - c[11]};
    float pp[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) pp[i] = c[3 * i] * e[0] + c[3 * i + 1] * e[1] + c[3 * i + 2] * e[2];
    // the reference divides by p.z and negates v only; the pinhole projection (pixel_aligned) negates both before that
    float u = pp[0] / pp[2] / scale, v = pp[1] / pp[2] / scale;
    if (pixel_aligned) u = -u;
    else v = -v;
    float ix = (u + 1.f) * 0.5f * (float)(fw - 1), iy = (v + 1.f) * 0.5f * (float)(fh - 1);
    ix = fminf(fmaxf(ix, 0.f), (float)(fw - 1));
    iy = fminf(fmaxf(iy, 0.f), (float)(fh - 1));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0, x1 = min(x0 + 1, (int)fw - 1), y1 = min(y0 + 1, (int)fh - 1);
    const float wx = ix - fx0, wy = iy - fy0;
    const int b = (int)(k * fh * fw);
    auto off = [&](int yy, int xx) { return (b + yy * (int)fw + xx) * (int)WIDTH; };
    taps[q] = make_int4(off(y0, x0), off(y0, x1), off(y1, x0), off(y1, x1));
    tapw[q] = make_float4((1.f - wx) * (1.f - wy), wx * (1.f - wy), (1.f - wx) * wy, wx * wy);
}

// Network.py:5-11 + :73-77: [x, sin(2^i 1.5 x), cos(2^i 1.5 x) for i < 6, d / |d|] in fp32 -> fp16, columns 42..63 zero.
__global__ void pn_encode_kernel(uint32_t Ms, uint32_t S, const float* __restrict__ rays, const float* __restrict__ z, __half* __restrict__ enc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= Ms) return;
    const float* r = rays + (size_t)(j / S) * 6;
    const float zz = z[j % S];
    float col[ENC_PAD];
#pragma unroll
    for (uint32_t i = 0; i < ENC_PAD; ++i) col[i] = 0.f;
    float x[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) x[a] = col[a] = r[a] + r[3 + a] * zz;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float y = ldexpf(x[a], i) * 1.5f;
            col[3 + 6 * i + a] = sinf(y);
            col[6 + 6 * i + a] = cosf(y);
        }
    }
    const float n = fmaxf(sqrtf(r[3] * r[3] + r[4] * r[4] + r[5] * r[5]), 1e-12f);
#pragma unroll
    for (int a = 0; a < 3; ++a) col[ENC_COLS - 3 + a] = r[3 + a] / n;
    uint4* o = reinterpret_cast<uint4*>(enc + (size_t)j * ENC_PAD);
#pragma unroll
    for (uint32_t g = 0; g < ENC_PAD / 8; ++g)
        o[g] = make_uint4(wg::pack_half2(col[8 * g], col[8 * g + 1]), wg::pack_half2(col[8 * g + 2], col[8 * g + 3]),
                          wg::pack_half2(col[8 * g + 4], col[8 * g + 5]), wg::pack_half2(col[8 * g + 6], col[8 * g + 7]));
}

// Network.py:86: the mean over references, summed in reference order in fp32.
__global__ void pn_mean_kernel(uint32_t Ms, uint32_t n_ref, const __half2* __restrict__ f, __half2* __restrict__ mean) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, per = (size_t)Ms * WIDTH / 2;
    if (i >= per) return;
    float2 s = make_float2(0.f, 0.f);
    for (uint32_t k = 0; k < n_ref; ++k) {
        const float2 v = __half22float2(f[k * per + i]);
        s.x += v.x;
        s.y += v.y;
    }
    mean[i] = __floats2half2_rn(s.x / (float)n_ref, s.y / (float)n_ref);
}

// Backward of the mean into the last f1 block's output ReLU: dr[k Ms + j] = dmean[j] / n_ref where r > 0.
__global__ void pn_mean_bwd_kernel(uint32_t Ms, uint32_t n_ref, const __half* __restrict__ dmean, const __half* __restrict__ r,
                                   __half* __restrict__ dr) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, per = (size_t)Ms * WIDTH;
    if (i >= per * n_ref) return;
    const float v = __half2float(dmean[i % per]) * (1.f / (float)n_ref);
    dr[i] = __hgt(r[i], __float2half(0.f)) ? __float2half_rn(v) : __float2half(0.f);
}

// Backward of the stem broadcast: ds[j] = sum_k dx[k Ms + j] (reference order, fp32) where the stem output s > 0.
__global__ void pn_stem_bwd_kernel(uint32_t Ms, uint32_t n_ref, const __half* __restrict__ dx, const __half* __restrict__ s, __half* __restrict__ ds) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, per = (size_t)Ms * WIDTH;
    if (i >= per) return;
    float a = 0.f;
    for (uint32_t k = 0; k < n_ref; ++k) a += __half2float(dx[k * per + i]);
    ds[i] = __hgt(s[i], __float2half(0.f)) ? __float2half_rn(a) : __float2half(0.f);
}

// Backward of Network.py:92-93: d(final_layer output) from d(raw) and raw = (relu(o0), sigmoid(o1:4)); (Ms, 8), columns 4..7 zero.
__global__ void pn_head_bwd_kernel(uint32_t Ms, const __half* __restrict__ raw, const __half* __restrict__ draw, __half* __restrict__ dpre) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= Ms) return;
    float o[4];
    o[0] = __half2float(raw[4 * (size_t)j]) > 0.f ? __half2float(draw[4 * (size_t)j]) : 0.f;
#pragma unroll
    for (int c = 1; c < 4; ++c) {
        const float y = __half2float(raw[4 * (size_t)j + c]);
        o[c] = __half2float(draw[4 * (size_t)j + c]) * y * (1.f - y);
    }
    *reinterpret_cast<uint4*>(dpre + (size_t)j * HEAD_PAD) = make_uint4(wg::pack_half2(o[0], o[1]), wg::pack_half2(o[2], o[3]), 0u, 0u);
}

// Bias gradients: column sums of the first `cols` (even) columns of dy (rows, ld) over CS_CHUNKS fixed row chunks -> part (CS_CHUNKS, cols).
__global__ void pn_colsum_kernel(uint32_t rows, uint32_t cols, uint32_t ld, const __half* __restrict__ dy, float* __restrict__ part) {
    const uint32_t c = 2 * threadIdx.x;
    if (c >= cols) return;
    const uint32_t r0 = (uint32_t)((uint64_t)rows * blockIdx.x / gridDim.x), r1 = (uint32_t)((uint64_t)rows * (blockIdx.x + 1) / gridDim.x);
    float2 s = make_float2(0.f, 0.f);
    for (uint32_t r = r0; r < r1; ++r) {
        const float2 v = __half22float2(*reinterpret_cast<const __half2*>(dy + (size_t)r * ld + c));
        s.x += v.x;
        s.y += v.y;
    }
    part[(size_t)blockIdx.x * cols + c] = s.x;
    part[(size_t)blockIdx.x * cols + c + 1] = s.y;
}

// out[i] = sum of part[z][i] over z in order: the partial sums of the wgrad and bias-gradient chunks.
__global__ void pn_reduce_kernel(uint32_t count, uint32_t chunks, const float* __restrict__ part, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    float s = 0.f;
    for (uint32_t z = 0; z < chunks; ++z) s += part[(size_t)z * count + i];
    out[i] = s;
}

// ---- composite (Render.py:16-18, :34-46), one warp a ray, samples 2 lane and 2 lane + 1 ------------------------------------------------
struct RaySamples {
    float sig[2], c[2][3], delta[2], e[2], tt[2], T[2], w[2];
};

__device__ __forceinline__ void composite_ray(uint32_t ray, uint32_t S, const __half* raw, const float* z, const float* rays, uint32_t lane,
                                              RaySamples& a) {
    const float* r = rays + (size_t)ray * 6;
    const float dn = sqrtf(r[3] * r[3] + r[4] * r[4] + r[5] * r[5]);
    float local = 1.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t i = 2 * lane + h;
        a.sig[h] = 0.f;
        a.c[h][0] = a.c[h][1] = a.c[h][2] = 0.f;
        a.delta[h] = 0.f;
        if (i < S) {
            const __half* q = raw + ((size_t)ray * S + i) * 4;
            a.sig[h] = __half2float(q[0]);
            for (int ch = 0; ch < 3; ++ch) a.c[h][ch] = __half2float(q[1 + ch]);
            a.delta[h] = (i + 1 < S ? z[i + 1] - z[i] : 1e10f) * dn;
        }
        a.e[h] = expf(-a.sig[h] * a.delta[h]);
        const float alpha = 1.f - a.e[h];
        a.tt[h] = i < S ? 1.f - alpha + 1e-7f : 1.f;
        a.w[h] = alpha;                         // times T below
        local *= a.tt[h];
    }
    // exclusive product scan of the lanes' (t_a t_b): the transmittance cumprod([1, 1 - alpha + 1e-7])
    float inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (uint32_t)o) inc *= v;
    }
    float ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = 1.f;
    a.T[0] = ex;
    a.T[1] = ex * a.tt[0];
    for (int h = 0; h < 2; ++h) a.w[h] = 2 * lane + h < S ? a.w[h] * a.T[h] : 0.f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void pn_composite_fwd_kernel(uint32_t R, uint32_t S, const __half* __restrict__ raw, const float* __restrict__ z,
                                        const float* __restrict__ rays, float* __restrict__ rgb, float* __restrict__ depth, float* __restrict__ acc) {
    const uint32_t ray = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
    if (ray >= R) return;
    RaySamples a;
    composite_ray(ray, S, raw, z, rays, lane, a);
    float c3[3], dz = 0.f;
    for (int ch = 0; ch < 3; ++ch) c3[ch] = warp_sum(a.w[0] * a.c[0][ch] + a.w[1] * a.c[1][ch]);
    for (int h = 0; h < 2; ++h)
        if (2 * lane + h < S) dz += a.w[h] * z[2 * lane + h];
    dz = warp_sum(dz);
    const float ac = warp_sum(a.w[0] + a.w[1]);
    if (lane == 0) {
        for (int ch = 0; ch < 3; ++ch) rgb[3 * (size_t)ray + ch] = c3[ch];
        if (depth) depth[ray] = dz;
        if (acc) acc[ray] = ac;
    }
}

// MSE over the 3 R colour entries (main.py:33, :45) and grad_scale * dloss / draw, saturated to the fp16 range.
__global__ void pn_composite_loss_bwd_kernel(uint32_t R, uint32_t S, const __half* __restrict__ raw, const float* __restrict__ z,
                                             const float* __restrict__ rays, const float* __restrict__ target, float grad_scale,
                                             float* __restrict__ rgb, float* __restrict__ loss, __half* __restrict__ draw) {
    const uint32_t ray = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
    if (ray >= R) return;
    RaySamples a;
    composite_ray(ray, S, raw, z, rays, lane, a);
    float g[3], l = 0.f;
    for (int ch = 0; ch < 3; ++ch) {
        const float c = warp_sum(a.w[0] * a.c[0][ch] + a.w[1] * a.c[1][ch]);
        const float diff = c - target[3 * (size_t)ray + ch];
        l += diff * diff;
        g[ch] = grad_scale * 2.f * diff / (3.f * (float)R);
        if (lane == 0 && rgb) rgb[3 * (size_t)ray + ch] = c;
    }
    if (lane == 0 && loss) loss[ray] = l / (3.f * (float)R);
    float gc[2], wgc[2];
    for (int h = 0; h < 2; ++h) {
        gc[h] = g[0] * a.c[h][0] + g[1] * a.c[h][1] + g[2] * a.c[h][2];
        wgc[h] = a.w[h] * gc[h];
    }
    // exclusive suffix sum over later samples: S_i = sum_{k > i} w_k (g . c_k)
    float inc = wgc[0] + wgc[1];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_down_sync(0xffffffffu, inc, o);
        if (lane + o < 32) inc += v;
    }
    float ex = __shfl_down_sync(0xffffffffu, inc, 1);
    if (lane == 31) ex = 0.f;
    const float suf[2] = {ex + wgc[1], ex};
    for (int h = 0; h < 2; ++h) {
        const uint32_t i = 2 * lane + h;
        if (i >= S) continue;
        const float dalpha = a.T[h] * gc[h] - suf[h] / a.tt[h];
        const float ds = dalpha * a.delta[h] * a.e[h];
        auto sat = [](float v) { return __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f)); };
        __half* o = draw + ((size_t)ray * S + i) * 4;
        o[0] = sat(ds);
        for (int ch = 0; ch < 3; ++ch) o[1 + ch] = sat(a.w[h] * g[ch]);
    }
}

// ---- host ------------------------------------------------------------------------------------------------------------------------------
struct Buf {
    size_t off = 0;
    size_t take(size_t bytes) {
        const size_t o = off;
        off += (bytes + 255) & ~(size_t)255;
        return o;
    }
};

// Offsets of the forward's buffers.  train: every activation the backward reads has its own buffer; inference: the blocks share them.
struct FwdLayout {
    size_t enc, taps, tapw, s, tmp, mean, f1_g[N_F1], f1_x[N_F1], f1_h[N_F1], f1_r[N_F1], f2_h[N_F2], f2_r[N_F2], f2_out[N_F2], bytes;
    bool train;
    FwdLayout(uint32_t Ms, uint32_t n_ref, bool tr) : train(tr) {
        const size_t M3 = (size_t)Ms * n_ref, big = M3 * WIDTH * 2, small = (size_t)Ms * WIDTH * 2;
        Buf b;
        enc = b.take((size_t)Ms * ENC_PAD * 2);
        taps = b.take(M3 * 16);
        tapw = b.take(M3 * 16);
        s = b.take(small);
        tmp = b.take(big);
        mean = b.take(small);
        const size_t x0 = b.take(big), h0 = b.take(big);
        for (uint32_t i = 0; i < N_F1; ++i) {
            f1_x[i] = i == 0 || !tr ? x0 : b.take(big);
            f1_h[i] = i == 0 || !tr ? h0 : b.take(big);
            f1_g[i] = tr ? b.take(big) : SIZE_MAX;
            f1_r[i] = tr ? b.take(big) : SIZE_MAX;
        }
        for (uint32_t i = 0; i < N_F2; ++i) {
            f2_h[i] = tr ? b.take(small) : h0;
            f2_r[i] = tr ? b.take(small) : SIZE_MAX;
            f2_out[i] = tr ? b.take(small) : mean;
        }
        bytes = b.off;
    }
};

struct BwdLayout {
    size_t dr, dh, dx, dg, dmean, dpre, wpart, cpart, bytes;
    BwdLayout(uint32_t Ms, uint32_t n_ref) {
        const size_t big = (size_t)Ms * n_ref * WIDTH * 2;
        Buf b;
        dr = b.take(big);
        dh = b.take(big);
        dx = b.take(big);
        dg = b.take(big);
        dmean = b.take((size_t)Ms * WIDTH * 2);
        dpre = b.take((size_t)Ms * HEAD_PAD * 2);
        wpart = b.take((size_t)WG_CHUNKS * WIDTH * WIDTH * 4);
        cpart = b.take((size_t)CS_CHUNKS * WIDTH * 4);
        bytes = b.off;
    }
};

template <int EPI>
int launch_gemm(cudaStream_t st, const GemmArgs& a, uint32_t z = 1) {
    if (a.M == 0 || a.N == 0) return 0;
    if (ngp_first_use((const void*)pn_gemm_kernel<EPI>))
        NGP_CHECK_CUDA(cudaFuncSetAttribute(pn_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM));
    const dim3 grid((a.N + BN - 1) / BN, (a.M + BM - 1) / BM, z);
    pn_gemm_kernel<EPI><<<grid, THREADS, GEMM_SMEM, st>>>(a);
    NGP_LAUNCH_CHECK();
    return 0;
}

inline GemmArgs gemm(const __half* A, uint32_t lda, const __half* B, uint32_t ldb, uint32_t M, uint32_t N, uint32_t K) {
    GemmArgs a{};
    a.A = A;
    a.B = B;
    a.lda = lda;
    a.ldb = ldb;
    a.M = M;
    a.N = N;
    a.K = K;
    a.kb_lim = K;
    a.ldo = N;
    a.res_rows = M;
    a.res_scale = 1.f;
    return a;
}

#define PN_TRY(x)                 \
    do {                          \
        const int _r = (x);       \
        if (_r) return _r;        \
    } while (0)

// dW (rows x cols, fp32, into grad) = dy^T x over `n` rows, and the bias gradient (rows) = column sums of dy.
int wgrad(cudaStream_t st, const __half* dy, uint32_t ldy, const __half* x, uint32_t ldx, uint32_t n, uint32_t rows, uint32_t cols, const Gather* g,
          float* wpart, float* cpart, float* grad_w, float* grad_b) {
    GemmArgs a = gemm(dy, ldy, x, ldx, rows, cols, n);
    a.part = wpart;
    if (g) {
        a.gather_b = 1;
        a.g = *g;
    }
    PN_TRY(launch_gemm<EPI_WGRAD>(st, a, WG_CHUNKS));
    pn_reduce_kernel<<<(rows * cols + 255) / 256, 256, 0, st>>>(rows * cols, WG_CHUNKS, wpart, grad_w);
    NGP_LAUNCH_CHECK();
    pn_colsum_kernel<<<CS_CHUNKS, (rows + 1) / 2, 0, st>>>(n, rows, ldy, dy, cpart);
    NGP_LAUNCH_CHECK();
    pn_reduce_kernel<<<(rows + 255) / 256, 256, 0, st>>>(rows, CS_CHUNKS, cpart, grad_b);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // namespace pn

using namespace pn;

extern "C" {

int ngp_pixelnerf_param_count(uint64_t* count_out) {
    *count_out = N_PARAMS;
    return 0;
}

int ngp_pixelnerf_workspace_bytes(uint32_t n_ref, uint32_t n_rows, uint64_t* saved_bytes, uint64_t* infer_bytes, uint64_t* bwd_bytes) {
    NGP_REQUIRE(n_ref >= 1, "ngp_pixelnerf_workspace_bytes: n_ref must be >= 1");
    if (saved_bytes) *saved_bytes = FwdLayout(n_rows, n_ref, true).bytes;
    if (infer_bytes) *infer_bytes = FwdLayout(n_rows, n_ref, false).bytes;
    if (bwd_bytes) *bwd_bytes = BwdLayout(n_rows, n_ref).bytes;
    return 0;
}

int ngp_pixelnerf_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* z, const void* params, const void* feats,
                      uint32_t n_ref, uint32_t feat_h, uint32_t feat_w, const float* cams, float scale, int pixel_aligned, void* raw_out, void* saved,
                      void* scratch) {
    NGP_REQUIRE(n_samples > 0 && n_ref >= 1 && feat_h >= 1 && feat_w >= 1, "ngp_pixelnerf_fwd: n_samples, n_ref and the feature size must be > 0");
    const uint64_t Ms64 = (uint64_t)n_rays * n_samples;
    NGP_REQUIRE(Ms64 * n_ref * WIDTH < (1ull << 40) && Ms64 * n_ref < (1ull << 31) && (uint64_t)n_ref * feat_h * feat_w * WIDTH < (1ull << 31),
                "ngp_pixelnerf_fwd: too many rows or feature texels");
    // the GEMMs put 128-row tiles on grid.y, which stops at 65535
    NGP_REQUIRE(Ms64 * n_ref <= 65535ull * BM, "ngp_pixelnerf_fwd: at most 8 388 480 reference rows (n_rays * n_samples * n_ref) a call");
    const uint32_t Ms = (uint32_t)Ms64, M3 = Ms * n_ref;
    if (Ms == 0) return 0;
    void* ws = saved ? saved : scratch;
    NGP_REQUIRE(rays && z && params && feats && cams && raw_out && ws, "ngp_pixelnerf_fwd: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)feats & 15) == 0 && ((uintptr_t)ws & 255) == 0, "ngp_pixelnerf_fwd: misaligned buffer");
    cudaStream_t st = (cudaStream_t)stream;
    const FwdLayout L(Ms, n_ref, saved != nullptr);
    uint8_t* w8 = (uint8_t*)ws;
    auto H = [&](size_t off) { return off == SIZE_MAX ? (__half*)nullptr : (__half*)(w8 + off); };
    const __half* P = (const __half*)params;
    int4* taps = (int4*)(w8 + L.taps);
    float4* tapw = (float4*)(w8 + L.tapw);
    pn_taps_kernel<<<(M3 + 255) / 256, 256, 0, st>>>(Ms, n_samples, n_ref, rays, z, cams, feat_h, feat_w, scale, pixel_aligned, taps, tapw);
    NGP_LAUNCH_CHECK();
    pn_encode_kernel<<<(Ms + 127) / 128, 128, 0, st>>>(Ms, n_samples, rays, z, H(L.enc));
    NGP_LAUNCH_CHECK();
    // stem: s = relu(W enc + b), once per sample
    GemmArgs a = gemm(H(L.enc), ENC_PAD, P + P_STEM, ENC_PAD, Ms, WIDTH, ENC_PAD);
    a.bias = P + P_STEM + WIDTH * ENC_PAD;
    a.out0 = H(L.s);
    PN_TRY(launch_gemm<EPI_FWD>(st, a));
    const Gather g{taps, tapw, (const __half*)feats};
    for (uint32_t i = 0; i < N_F1; ++i) {
        const __half* blk = P + P_F1 + i * 3 * LIN;
        // x = res + relu(W_img feat + b): res is the stem output broadcast over the references, then the previous block's output
        a = gemm(nullptr, 0, blk, WIDTH, M3, WIDTH, WIDTH);
        a.gather_a = 1;
        a.g = g;
        a.bias = blk + WIDTH * WIDTH;
        a.out0 = H(L.f1_g[i]);
        a.res = i == 0 ? H(L.s) : H(L.tmp);
        a.res_rows = i == 0 ? Ms : M3;
        a.out1 = H(L.f1_x[i]);
        PN_TRY(launch_gemm<EPI_FWD>(st, a));
        a = gemm(H(L.f1_x[i]), WIDTH, blk + LIN, WIDTH, M3, WIDTH, WIDTH);
        a.bias = blk + LIN + WIDTH * WIDTH;
        a.out0 = H(L.f1_h[i]);
        PN_TRY(launch_gemm<EPI_FWD>(st, a));
        a = gemm(H(L.f1_h[i]), WIDTH, blk + 2 * LIN, WIDTH, M3, WIDTH, WIDTH);
        a.bias = blk + 2 * LIN + WIDTH * WIDTH;
        a.out0 = H(L.f1_r[i]);
        a.res = H(L.f1_x[i]);
        a.out1 = H(L.tmp);
        PN_TRY(launch_gemm<EPI_FWD>(st, a));
    }
    pn_mean_kernel<<<(uint32_t)(((size_t)Ms * WIDTH / 2 + 255) / 256), 256, 0, st>>>(Ms, n_ref, (const __half2*)H(L.tmp), (__half2*)H(L.mean));
    NGP_LAUNCH_CHECK();
    const __half* x = H(L.mean);
    for (uint32_t i = 0; i < N_F2; ++i) {
        const __half* blk = P + P_F2 + i * 2 * LIN;
        a = gemm(x, WIDTH, blk, WIDTH, Ms, WIDTH, WIDTH);
        a.bias = blk + WIDTH * WIDTH;
        a.out0 = H(L.f2_h[i]);
        PN_TRY(launch_gemm<EPI_FWD>(st, a));
        a = gemm(H(L.f2_h[i]), WIDTH, blk + LIN, WIDTH, Ms, WIDTH, WIDTH);
        a.bias = blk + LIN + WIDTH * WIDTH;
        a.out0 = H(L.f2_r[i]);
        a.res = x;
        a.out1 = H(L.f2_out[i]);
        PN_TRY(launch_gemm<EPI_FWD>(st, a));
        x = H(L.f2_out[i]);
    }
    a = gemm(x, WIDTH, P + P_HEAD, WIDTH, Ms, 4, WIDTH);
    a.bias = P + P_HEAD + 4 * WIDTH;
    a.out0 = (__half*)raw_out;
    return launch_gemm<EPI_HEAD>(st, a);
}

int ngp_pixelnerf_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, uint32_t n_ref, const void* params, const void* feats, const void* saved,
                      const void* raw, const void* draw, void* scratch, float* grad) {
    NGP_REQUIRE(n_samples > 0 && n_ref >= 1, "ngp_pixelnerf_bwd: n_samples and n_ref must be > 0");
    NGP_REQUIRE((uint64_t)n_rays * n_samples * n_ref <= 65535ull * BM, "ngp_pixelnerf_bwd: at most 8 388 480 reference rows a call");
    const uint32_t Ms = n_rays * n_samples, M3 = Ms * n_ref;
    NGP_REQUIRE(params && feats && saved && raw && draw && scratch && grad, "ngp_pixelnerf_bwd: NULL input");
    NGP_REQUIRE(((uintptr_t)saved & 255) == 0 && ((uintptr_t)scratch & 255) == 0 && ((uintptr_t)params & 15) == 0, "ngp_pixelnerf_bwd: misaligned buffer");
    cudaStream_t st = (cudaStream_t)stream;
    if (Ms == 0) {
        NGP_CHECK_CUDA(cudaMemsetAsync(grad, 0, (size_t)N_PARAMS * 4, st));
        return 0;
    }
    const FwdLayout L(Ms, n_ref, true);
    const BwdLayout B(Ms, n_ref);
    const uint8_t* s8 = (const uint8_t*)saved;
    uint8_t* w8 = (uint8_t*)scratch;
    auto S_ = [&](size_t off) { return (const __half*)(s8 + off); };
    auto W_ = [&](size_t off) { return (__half*)(w8 + off); };
    const __half* P = (const __half*)params;
    float* wpart = (float*)(w8 + B.wpart);
    float* cpart = (float*)(w8 + B.cpart);
    __half *dr = W_(B.dr), *dh = W_(B.dh), *dx = W_(B.dx), *dg = W_(B.dg), *dpre = W_(B.dpre), *dmean = W_(B.dmean);
    const Gather g{(const int4*)(s8 + L.taps), (const float4*)(s8 + L.tapw), (const __half*)feats};
    // the pad columns 42..63 of the stem weight get exact zeros from the zero encoding columns; the flat gradient has no other gaps
    pn_head_bwd_kernel<<<(Ms + 127) / 128, 128, 0, st>>>(Ms, (const __half*)raw, (const __half*)draw, dpre);
    NGP_LAUNCH_CHECK();
    const __half* x_head = S_(L.f2_out[N_F2 - 1]);
    PN_TRY(wgrad(st, dpre, HEAD_PAD, x_head, WIDTH, Ms, 4, WIDTH, nullptr, wpart, cpart, grad + P_HEAD, grad + P_HEAD + 4 * WIDTH));
    // dx_head = dpre W_head: the last f2 block's output gradient (dx) and its r-masked part (dr)
    GemmArgs a = gemm(dpre, HEAD_PAD, P + P_HEAD, WIDTH, Ms, WIDTH, HEAD_PAD);
    a.kb_lim = 4;
    a.out0 = dx;
    a.out2 = dr;
    a.mask2 = S_(L.f2_r[N_F2 - 1]);
    PN_TRY(launch_gemm<EPI_BWD>(st, a));
    for (int i = N_F2 - 1; i >= 0; --i) {
        const __half* blk = P + P_F2 + i * 2 * LIN;
        float* gb = grad + P_F2 + i * 2 * LIN;
        const __half* xin = i == 0 ? S_(L.mean) : S_(L.f2_out[i - 1]);
        a = gemm(dr, WIDTH, blk + LIN, WIDTH, Ms, WIDTH, WIDTH);
        a.out1 = dh;
        a.mask1 = S_(L.f2_h[i]);
        PN_TRY(launch_gemm<EPI_BWD>(st, a));
        PN_TRY(wgrad(st, dr, WIDTH, S_(L.f2_h[i]), WIDTH, Ms, WIDTH, WIDTH, nullptr, wpart, cpart, gb + LIN, gb + LIN + WIDTH * WIDTH));
        a = gemm(dh, WIDTH, blk, WIDTH, Ms, WIDTH, WIDTH);
        a.res = dx;
        a.out0 = i == 0 ? dmean : dx;      // d(mean) is read broadcast while the last f1 block writes dx: its own buffer
        if (i > 0) {
            a.out2 = dr;
            a.mask2 = S_(L.f2_r[i - 1]);
        }
        PN_TRY(launch_gemm<EPI_BWD>(st, a));
        PN_TRY(wgrad(st, dh, WIDTH, xin, WIDTH, Ms, WIDTH, WIDTH, nullptr, wpart, cpart, gb, gb + WIDTH * WIDTH));
    }
    // d(mean), split into n_ref equal parts for the last f1 block
    pn_mean_bwd_kernel<<<(uint32_t)(((size_t)M3 * WIDTH + 255) / 256), 256, 0, st>>>(Ms, n_ref, dmean, S_(L.f1_r[N_F1 - 1]), dr);
    NGP_LAUNCH_CHECK();
    for (int i = N_F1 - 1; i >= 0; --i) {
        const __half* blk = P + P_F1 + i * 3 * LIN;
        float* gb = grad + P_F1 + i * 3 * LIN;
        a = gemm(dr, WIDTH, blk + 2 * LIN, WIDTH, M3, WIDTH, WIDTH);
        a.out1 = dh;
        a.mask1 = S_(L.f1_h[i]);
        PN_TRY(launch_gemm<EPI_BWD>(st, a));
        PN_TRY(wgrad(st, dr, WIDTH, S_(L.f1_h[i]), WIDTH, M3, WIDTH, WIDTH, nullptr, wpart, cpart, gb + 2 * LIN, gb + 2 * LIN + WIDTH * WIDTH));
        // dx = dh W1 + dout; dout is d(mean) / n_ref broadcast for the last block, the next block's dx otherwise
        a = gemm(dh, WIDTH, blk + LIN, WIDTH, M3, WIDTH, WIDTH);
        a.res = dx;
        if (i == (int)N_F1 - 1) {
            a.res = dmean;
            a.res_rows = Ms;
            a.res_scale = 1.f / (float)n_ref;
        }
        a.out0 = dx;
        a.out1 = dg;
        a.mask1 = S_(L.f1_g[i]);
        if (i > 0) {
            a.out2 = dr;
            a.mask2 = S_(L.f1_r[i - 1]);
        }
        PN_TRY(launch_gemm<EPI_BWD>(st, a));
        PN_TRY(wgrad(st, dh, WIDTH, S_(L.f1_x[i]), WIDTH, M3, WIDTH, WIDTH, nullptr, wpart, cpart, gb + LIN, gb + LIN + WIDTH * WIDTH));
        PN_TRY(wgrad(st, dg, WIDTH, nullptr, WIDTH, M3, WIDTH, WIDTH, &g, wpart, cpart, gb, gb + WIDTH * WIDTH));
    }
    pn_stem_bwd_kernel<<<(uint32_t)(((size_t)Ms * WIDTH + 255) / 256), 256, 0, st>>>(Ms, n_ref, dx, S_(L.s), dh);
    NGP_LAUNCH_CHECK();
    return wgrad(st, dh, WIDTH, S_(L.enc), ENC_PAD, Ms, WIDTH, ENC_PAD, nullptr, wpart, cpart, grad + P_STEM, grad + P_STEM + WIDTH * ENC_PAD);
}

int ngp_pixelnerf_composite_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, const float* z, const float* rays, float* rgb_out,
                                float* depth_out, float* acc_out) {
    NGP_REQUIRE(n_samples >= 1 && n_samples <= 64, "ngp_pixelnerf_composite_fwd: n_samples must be in [1, 64]");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(raw && z && rays && rgb_out, "ngp_pixelnerf_composite_fwd: NULL input");
    pn_composite_fwd_kernel<<<(n_rays + 7) / 8, 256, 0, (cudaStream_t)stream>>>(n_rays, n_samples, (const __half*)raw, z, rays, rgb_out, depth_out,
                                                                               acc_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_pixelnerf_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, const float* z, const float* rays,
                                     const float* target, float grad_scale, float* rgb_out, float* loss_out, void* draw_out) {
    NGP_REQUIRE(n_samples >= 1 && n_samples <= 64, "ngp_pixelnerf_composite_loss_bwd: n_samples must be in [1, 64]");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(raw && z && rays && target && draw_out, "ngp_pixelnerf_composite_loss_bwd: NULL input");
    pn_composite_loss_bwd_kernel<<<(n_rays + 7) / 8, 256, 0, (cudaStream_t)stream>>>(n_rays, n_samples, (const __half*)raw, z, rays, target,
                                                                                    grad_scale, rgb_out, loss_out, (__half*)draw_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
