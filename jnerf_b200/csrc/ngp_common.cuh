// Shared host/device helpers for libngp_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string>

// ---- error plumbing -----------------------------------------------------------------------------
void ngp_set_error(const std::string& msg);
#define NGP_CHECK_CUDA(expr)                                                                          \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess) {                                                                      \
            ngp_set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                        \
            return 1;                                                                                 \
        }                                                                                             \
    } while (0)
#define NGP_REQUIRE(cond, msg)                                                                        \
    do {                                                                                              \
        if (!(cond)) {                                                                                \
            ngp_set_error(std::string(msg));                                                          \
            return 2;                                                                                 \
        }                                                                                             \
    } while (0)
#define NGP_LAUNCH_CHECK() NGP_CHECK_CUDA(cudaGetLastError())

int ngp_num_sms();
// 128-byte TMA descriptor (CUtensorMap) of a row-major (n_rows, 32) fp16 matrix with an 8-column x 128-row box; false = no driver support
struct alignas(64) NgpTensorMap { unsigned long long opaque[16]; };
bool ngp_make_rows32_tensormap(NgpTensorMap* out, const void* base, unsigned long long n_rows);
bool ngp_first_use(const void* kernel);      // true the first time a kernel is seen on the current device (one-time attribute setup)

// ---- fire-and-forget reductions --------------------------------------------------------------------
// atomicAdd(__half2*) on a generic pointer compiles to QSPC + ATOM (returning a predicate) + a CAS spin fallback, i.e. every
// reduction waits for its round trip.  With the address converted to the global window the same operation is a single
// RED.E.ADD.F16x2 that retires at issue (HashEncode.h:339-347 only needs the sum, never the old value).
__device__ __forceinline__ void red_add_h2(__half2* addr, float a, float b) {
    const __half2 v = __floats2half2_rn(a, b);
    asm volatile("red.global.add.noftz.f16x2 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "r"(*reinterpret_cast<const uint32_t*>(&v)) : "memory");
}
// two neighbouring f16x2 entries (one aligned 8-byte word) in one request: REDG.E.ADD.F16x4
__device__ __forceinline__ void red_add_h2x2(__half2* addr8, float a0, float b0, float a1, float b1) {
    const __half2 v0 = __floats2half2_rn(a0, b0), v1 = __floats2half2_rn(a1, b1);
    asm volatile("red.global.add.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(__cvta_generic_to_global(addr8)), "r"(*reinterpret_cast<const uint32_t*>(&v0)),
                 "r"(*reinterpret_cast<const uint32_t*>(&v1)) : "memory");
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_f2(float2* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(__cvta_generic_to_global(addr)), "f"(a), "f"(b) : "memory");
}

// ---- hash-grid level record (R1) ------------------------------------------------------------------
struct __align__(32) NgpLevel {
    float scale;          // exp2f(level*log2_pls)*base - 1        (HashEncode.h:149)
    uint32_t resolution;  // (uint32_t)ceil(scale) + 1              (HashEncode.h:151)
    uint32_t offset;      // first entry of the level
    uint32_t size;        // entries in the level (hashmap_size)
    uint32_t hashed;      // 1: prime-XOR hash, 0: dense stride index (HashEncode.h:74-94)
    uint32_t prime[3];    // get_index(p0,p1,p2) = p0*prime[0] ^ p1*prime[1] ^ p2*prime[2]  (cfg.hash_func, HE/hash_encoder.py:13-16)
};
static_assert(sizeof(NgpLevel) == 32, "NgpLevel must be 32 bytes");
constexpr int N_LEVELS = 16;

// Corner indices (entry index within the level) and trilinear weights of point x at one level.
// Index math is bit-exact w.r.t. grid_index/fast_hash (HashEncode.h:68-94) for coordinates that do not wrap
// uint32 (positions in [0,1], the sampler's contract).  Weight order = corner idx 0..7, bit d -> +1 in dim d.
__device__ __forceinline__ void hash_corners(const NgpLevel& lv, float x, float y, float z, uint32_t idx[8], float w[8]) {
    float px = fmaf(x, lv.scale, 0.5f), py = fmaf(y, lv.scale, 0.5f), pz = fmaf(z, lv.scale, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
    px -= fx; py -= fy; pz -= fz;
    const float wx[2] = {1.0f - px, px}, wy[2] = {1.0f - py, py}, wz[2] = {1.0f - pz, pz};
    if (lv.hashed) {
        const uint32_t mask = lv.size - 1;  // hashed levels always have size == 2^log2_hashmap_size
        const uint32_t hx0 = gx * lv.prime[0], hx1 = (gx + 1) * lv.prime[0];
        const uint32_t hy0 = gy * lv.prime[1], hy1 = (gy + 1) * lv.prime[1];
        const uint32_t hz0 = gz * lv.prime[2], hz1 = (gz + 1) * lv.prime[2];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const uint32_t hx = (c & 1) ? hx1 : hx0;
            const uint32_t hy = (c & 2) ? hy1 : hy0;
            const uint32_t hz = (c & 4) ? hz1 : hz0;
            idx[c] = (hx ^ hy ^ hz) & mask;
        }
    } else {
        const uint32_t res = lv.resolution, res2 = res * res;
        const uint32_t b = (gx + gy * res + gz * res2) % lv.size;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            uint32_t v = b + (c & 1) + ((c & 2) ? res : 0u) + ((c & 4) ? res2 : 0u);
            v -= (v >= lv.size) ? lv.size : 0u;
            idx[c] = v;
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) w[c] = (1.0f * wx[c & 1]) * wy[(c >> 1) & 1] * wz[(c >> 2) & 1];
}

// Split form used by the run-length kernels: cell coordinates + fractions, then indices of a cell, then weights.
struct HashCell {
    uint32_t gx, gy, gz;
    float fx, fy, fz;
};
__device__ __forceinline__ HashCell hash_cell(const NgpLevel& lv, float x, float y, float z) {
    HashCell c;
    float px = fmaf(x, lv.scale, 0.5f), py = fmaf(y, lv.scale, 0.5f), pz = fmaf(z, lv.scale, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    c.gx = (uint32_t)(int)fx; c.gy = (uint32_t)(int)fy; c.gz = (uint32_t)(int)fz;
    c.fx = px - fx; c.fy = py - fy; c.fz = pz - fz;
    return c;
}
__device__ __forceinline__ void hash_cell_indices(const NgpLevel& lv, uint32_t gx, uint32_t gy, uint32_t gz, uint32_t idx[8]) {
    if (lv.hashed) {
        const uint32_t mask = lv.size - 1;
        const uint32_t hx0 = gx * lv.prime[0], hx1 = (gx + 1) * lv.prime[0];
        const uint32_t hy0 = gy * lv.prime[1], hy1 = (gy + 1) * lv.prime[1];
        const uint32_t hz0 = gz * lv.prime[2], hz1 = (gz + 1) * lv.prime[2];
#pragma unroll
        for (int c = 0; c < 8; ++c) idx[c] = (((c & 1) ? hx1 : hx0) ^ ((c & 2) ? hy1 : hy0) ^ ((c & 4) ? hz1 : hz0)) & mask;
    } else {
        const uint32_t res = lv.resolution, res2 = res * res;
        const uint32_t b = (gx + gy * res + gz * res2) % lv.size;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            uint32_t v = b + (c & 1) + ((c & 2) ? res : 0u) + ((c & 4) ? res2 : 0u);
            v -= (v >= lv.size) ? lv.size : 0u;
            idx[c] = v;
        }
    }
}
// A full-occupancy scatter is bound by the number of L2 reduction REQUESTS (one per lane and instruction), not by bytes.  Corners c and
// c+1 of a cell are x-neighbours: whenever their entries share an aligned 8-byte word -- dense levels: even index; hashed levels:
// even x, because (x+1) ^ h = (x ^ h) ^ 1 then -- one REDG.F16x4 serves both.  Half of all cells qualify, i.e. 6 requests per cell
// instead of 8 on average; the sums formed are exactly the same.  Used by the standalone ngp_hash_bwd; the gather (64-bit loads) and
// the fused kernels do not use it.  The fused backward's 64-bit fixed-point scatter has no vector integer reduction to pair corners
// with (ptxas rejects red.global.add.v2.u64); it gives the features and x-neighbours of a cell to adjacent lanes of one instruction
// instead, so that one instruction addresses at most two 32-byte sectors per lane group (fused_net.cu, DESIGN.md section 4).
__device__ __forceinline__ void red_add_corners(__half2* __restrict__ g, const uint32_t idx[8], const float2 acc[8]) {
#pragma unroll
    for (int c = 0; c < 8; c += 2) {
        if ((idx[c] ^ idx[c + 1]) == 1u) {
            const bool lo = (idx[c] & 1u) == 0u;
            const float2 v0 = lo ? acc[c] : acc[c + 1], v1 = lo ? acc[c + 1] : acc[c];
            red_add_h2x2(g + (idx[c] & ~1u), v0.x, v0.y, v1.x, v1.y);
        } else {
            red_add_h2(g + idx[c], acc[c].x, acc[c].y);
            red_add_h2(g + idx[c + 1], acc[c + 1].x, acc[c + 1].y);
        }
    }
}
__device__ __forceinline__ void hash_cell_weights(const HashCell& c, float w[8]) {
    const float wx[2] = {1.0f - c.fx, c.fx}, wy[2] = {1.0f - c.fy, c.fy}, wz[2] = {1.0f - c.fz, c.fz};
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k] = (1.0f * wx[k & 1]) * wy[(k >> 1) & 1] * wz[(k >> 2) & 1];
}

// ---- SH degree 4 (SphericalEncode.h:65-95) ---------------------------------------------------------
__device__ __forceinline__ void sh4(float dx, float dy, float dz, float* o) {
    const float x = dx * 2.f - 1.f, y = dy * 2.f - 1.f, z = dz * 2.f - 1.f;
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// ---- pcg32 (ops/op_include/pcg32/pcg32.h) ----------------------------------------------------------
struct Pcg32 {
    uint64_t state, inc;
    __host__ __device__ uint32_t next_uint() {
        const uint64_t old = state;
        state = old * 0x5851f42d4c957f2dULL + inc;
        const uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
        const uint32_t rot = (uint32_t)(old >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
    }
    __host__ __device__ float next_float() {
        union { uint32_t u; float f; } x;
        x.u = (next_uint() >> 9) | 0x3f800000u;
        return x.f - 1.0f;
    }
    __host__ __device__ void advance(int64_t delta_) {
        uint64_t cur_mult = 0x5851f42d4c957f2dULL, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
        uint64_t delta = (uint64_t)delta_;
        while (delta > 0) {
            if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
            cur_plus = (cur_mult + 1) * cur_plus;
            cur_mult *= cur_mult;
            delta /= 2;
        }
        state = acc_mult * state + acc_plus;
    }
};

struct AdamArgs {
    float step_size, b1, b2, eps, decay, debias_old, debias_new, grad_scale;
};

// ---- morton (ray_sampler_header.h:642-667) ----------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu; v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u; v = (v * 0x00000005u) & 0x49249249u; return v;
}
__host__ __device__ __forceinline__ uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) {
    return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2);
}
__host__ __device__ __forceinline__ uint32_t morton3D_invert(uint32_t x) {
    x = x & 0x49249249; x = (x | (x >> 2)) & 0xc30c30c3; x = (x | (x >> 4)) & 0x0f00f00f;
    x = (x | (x >> 8)) & 0xff0000ff; x = (x | (x >> 16)) & 0x0000ffff; return x;
}

constexpr uint32_t NERF_GRIDSIZE = 128;
constexpr uint32_t NERF_GRID_N = NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE;
constexpr uint32_t NERF_STEPS = 1024;
__device__ __forceinline__ float nerf_min_cone() { return 1.73205080757f / 1024.0f; }
__device__ __forceinline__ float nerf_unwarp_dt(float dt, uint32_t cascades) {
    const float mn = nerf_min_cone();
    const float max_stepsize = mn * (float)(1u << (cascades - 1));
    return __fmaf_rn(dt, max_stepsize - mn, mn);   // calc_rgb.h:4-8 (a*b+c, contracted by nvcc in the reference build)
}
__device__ __forceinline__ float nerf_warp_dt(float dt, uint32_t cascades) {
    const float mn = nerf_min_cone();
    const float max_stepsize = mn * (float)(1u << (cascades - 1));
    return __fdiv_rn(__fsub_rn(dt, mn), __fsub_rn(max_stepsize, mn));
}
__device__ __forceinline__ float logistic_f(float x) { return 1.0f / (1.0f + expf(-x)); }
