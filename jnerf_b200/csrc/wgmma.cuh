// wgmma / TMA / mbarrier primitives for sm_90a (Hopper), written as inline PTX.
//
// Shared by the fully-fused MLP kernels (mlp_tc.cu, fused_net.cu).  The operand
// layout used everywhere is the un-swizzled ("interleave") canonical GMMA layout
// built from 8x16-byte core matrices, arranged as a *slab*:
//
//     slab[g][r][8 halfs]      g = feature group (8 features), r = row (0..127)
//     byte(r, f) = (f/8)*SLAB_GROUP_BYTES(rows) + r*16 + (f%8)*2
//
// Read as a K-major operand (rows = M/N index, features = K):  SBO = 128, LBO = rows*16.
// Read as an MN-major operand (features = M/N index, rows = K): SBO = rows*16, LBO = 128.
// The same bytes therefore feed the forward GEMM, the dgrad GEMM (weights
// transposed) and the wgrad GEMM (activations transposed) without any copy.
//
// A wgmma is issued by all 128 threads of a warpgroup (four consecutive warps, the first one a multiple of 4) and leaves
// D[64 x N] in registers: thread i of the warpgroup holds d[4c + 2h + j] = D[16*(i/32) + (i%32)/4 + 8h][8c + 2*(i%4) + j].
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- mbarrier -------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a descriptor mistake must not hang the GPU.  Returns false on timeout.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
#pragma unroll 1   // the compiler otherwise unrolls this spin loop dozens of times
    for (uint32_t spin = 0; spin < (1u << 22); ++spin) {
        if (mbar_try_wait(bar, parity)) return true;
    }
    return false;
}

// ---- fences ---------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
    // make generic-proxy st.shared visible to the async proxy (wgmma operand reads, TMA stores)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA (cp.async.bulk.tensor) -------------------------------------------------------------------
// A 2-D box of a row-major (rows, 32) fp16 matrix, 8 columns x 128 rows, lands in shared memory as [128 rows][8 halfs] = exactly one
// feature group of an operand slab (see the top of this file), so the encoded-feature rows kept for the backward pass travel
// HBM <-> slab as four tensor copies per 128-row tile instead of a 16-byte access per thread and group.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const void* tmap, uint32_t c0, uint32_t c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t c0, uint32_t c1, uint32_t src_smem) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(tmap), "r"(c0), "r"(c1), "r"(src_smem) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- descriptors ------------------------------------------------------------
// Shared-memory matrix descriptor, SWIZZLE_NONE (layout type 0, base offset 0).
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}

// ---- leader election -----------------------------------------------------------
// All 32 lanes of the warp must execute this convergently.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- warpgroup MMA ------------------------------------------------------------
// wgmma_fence before the first wgmma of a batch (orders the accumulator registers and the shared-memory operands written before
// it), then the wgmmas, wgmma_commit, and wgmma_wait<0> before the accumulators are read.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] B[16 x N], fp16 x fp16 -> fp32.  TA / TB: 0 = K-major operand, 1 = MN-major operand.
// acc = 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void mma_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void mma_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void mma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <uint32_t N, int TA, int TB>
__device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {
    static_assert(N == 16 || N == 32 || N == 64, "wgmma N");
    if constexpr (N == 16) mma_n16<TA, TB>(d, a, b, acc);
    else if constexpr (N == 32) mma_n32<TA, TB>(d, a, b, acc);
    else mma_n64<TA, TB>(d, a, b, acc);
}

// ---- slab helpers -----------------------------------------------------------
// K-major operand over a slab of `rows` rows starting at feature group g0, K block kb (16 features).
__device__ __forceinline__ uint64_t slab_desc_kmajor(uint32_t slab_saddr, uint32_t rows, uint32_t g0, uint32_t kb) {
    const uint32_t gb = rows * 16u;
    return smem_desc(slab_saddr + (g0 + 2u * kb) * gb, /*LBO*/ gb, /*SBO*/ 128u);
}
// MN-major operand: features [8*g0, ...) are the M/N index, rows are K; K block kb = rows [16kb,16kb+16).
__device__ __forceinline__ uint64_t slab_desc_mnmajor(uint32_t slab_saddr, uint32_t rows, uint32_t g0, uint32_t kb) {
    const uint32_t gb = rows * 16u;
    return smem_desc(slab_saddr + g0 * gb + kb * 256u, /*LBO*/ 128u, /*SBO*/ gb);
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace wg
