// R1-R4: hash-grid level table, standalone hash-grid forward/backward, SH encoder.
//
// Replaces the reference's 3-kernel forward (extract_position -> kernel_grid -> transpose_encoded_position,
// HE/op_header/HashEncode.h:36-50,117-252,254-268) and 3-step backward (transpose_gradients -> memset ->
// kernel_grid_backward, :270-284,299-396) with one kernel each:
//   * a warp covers 2 points x 16 levels, so the 32 half2 (or float2) features of a point are written /
//     read as one fully coalesced 64 B (128 B) row of the AoS (N,32) tensor -- no SoA scratch, no transposes;
//   * per-level {scale, resolution, offset, size, hashed} records are staged in shared memory once per CTA;
//   * each thread keeps PPT points in flight (8*PPT independent gathers) to cover L2/HBM latency.
// Algorithmic bytes (DESIGN.md): fwd 588 B/point fp16 (512 gather + 12 pos + 64 out), bwd 1100 B/point.
#include "ngp_common.cuh"
#include <cmath>
#include <cstdlib>

namespace {

__global__ void level_table_kernel(const uint32_t* __restrict__ offsets, int n_levels, uint32_t base_res, float log2_pls,
                                   NgpLevel* __restrict__ out, uint32_t p0, uint32_t p1, uint32_t p2) {
    const uint32_t level = threadIdx.x;
    if ((int)level >= n_levels) return;
    NgpLevel lv;
    lv.scale = exp2f(level * log2_pls) * base_res - 1.0f;          // HashEncode.h:149, evaluated on the device
    lv.resolution = ((uint32_t)ceil(lv.scale) + 1);                // :151
    lv.offset = offsets[level];
    lv.size = offsets[level + 1] - offsets[level];
    uint32_t stride = 1;                                            // grid_index loop, :80-91
    for (uint32_t dim = 0; dim < 3 && stride <= lv.size; ++dim) stride *= lv.resolution;
    lv.hashed = lv.size < stride ? 1u : 0u;
    lv.prime[0] = p0; lv.prime[1] = p1; lv.prime[2] = p2;
    out[level] = lv;
}

template <typename T> struct Vec2;
template <> struct Vec2<float> { using type = float2; };
template <> struct Vec2<__half> { using type = __half2; };

__device__ __forceinline__ float2 to_f2(float2 v) { return v; }
__device__ __forceinline__ float2 to_f2(__half2 v) { return __half22float2(v); }

constexpr int HASH_THREADS = 256;

__device__ __forceinline__ void red_add(__half2* addr, float a, float b) { red_add_h2(addr, a, b); }
__device__ __forceinline__ void red_add(float2* addr, float a, float b) { red_add_f2(addr, a, b); }

// ---- HashEncoder forward / backward (R2 / R3), run-length form -------------------------------------------------------------------
// Thread (level, sub) walks RUN consecutive points and keeps the 8 corner values (forward) / 8 fp32 corner accumulators (backward) of
// a grid cell while CONSECUTIVE points stay inside it -- the sampler hands points over ray-ordered, so at the coarse levels dozens
// do -- which cuts the L2 requests / f16x2 reductions by the mean run length.  Uniformly random points (no runs) gain nothing from it
// and lose little.  Per point the arithmetic is the reference's (corner order and fma chain of
// HashEncode.h:171-201); the backward rounds each run's fp32 sum once instead of once per point.
constexpr int RUN = 16;
constexpr int RUN_PTS_PER_BLOCK = (HASH_THREADS / N_LEVELS) * RUN;   // 256

template <typename T>
__global__ void __launch_bounds__(HASH_THREADS)
hash_fwd_kernel(uint32_t n, const float* __restrict__ x, const T* __restrict__ grid, const NgpLevel* __restrict__ levels,
                       T* __restrict__ out) {
    using V = typename Vec2<T>::type;
    __shared__ NgpLevel s_lv[N_LEVELS];
    if (threadIdx.x < N_LEVELS) s_lv[threadIdx.x] = levels[threadIdx.x];
    __syncthreads();
    const uint32_t level = threadIdx.x & (N_LEVELS - 1), sub = threadIdx.x / N_LEVELS;
    const NgpLevel lv = s_lv[level];
    const V* __restrict__ g = reinterpret_cast<const V*>(grid) + lv.offset;
    const uint32_t base = blockIdx.x * RUN_PTS_PER_BLOCK + sub * RUN;
    uint32_t cgx = 0xffffffffu, cgy = 0, cgz = 0;
    float2 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = make_float2(0.f, 0.f);
#pragma unroll 1
    for (int k = 0; k < RUN; ++k) {
        const uint32_t i = base + k;
        if (i >= n) break;
        const HashCell hc = hash_cell(lv, __ldg(x + 3 * (size_t)i), __ldg(x + 3 * (size_t)i + 1), __ldg(x + 3 * (size_t)i + 2));
        if (hc.gx != cgx || hc.gy != cgy || hc.gz != cgz) {
            cgx = hc.gx; cgy = hc.gy; cgz = hc.gz;
            uint32_t idx[8];
            hash_cell_indices(lv, cgx, cgy, cgz, idx);
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = to_f2(__ldg(g + idx[c]));   // (64-bit loads for x-neighbour pairs: 49 -> 52 us, not kept)
        }
        float w[8];
        hash_cell_weights(hc, w);
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) { a0 = fmaf(w[c], v[c].x, a0); a1 = fmaf(w[c], v[c].y, a1); }
        V r;
        if constexpr (sizeof(T) == 2) r = __floats2half2_rn(a0, a1); else r = make_float2(a0, a1);
        reinterpret_cast<V*>(out)[(size_t)i * N_LEVELS + level] = r;
    }
}

template <typename T>
__global__ void __launch_bounds__(HASH_THREADS)
hash_bwd_kernel(uint32_t n, const float* __restrict__ x, const T* __restrict__ dy, const NgpLevel* __restrict__ levels,
                       T* __restrict__ grid_grad) {
    using V = typename Vec2<T>::type;
    __shared__ NgpLevel s_lv[N_LEVELS];
    if (threadIdx.x < N_LEVELS) s_lv[threadIdx.x] = levels[threadIdx.x];
    __syncthreads();
    const uint32_t level = threadIdx.x & (N_LEVELS - 1), sub = threadIdx.x / N_LEVELS;
    const NgpLevel lv = s_lv[level];
    V* __restrict__ g = reinterpret_cast<V*>(grid_grad) + lv.offset;
    const uint32_t base = blockIdx.x * RUN_PTS_PER_BLOCK + sub * RUN;
    uint32_t cgx = 0xffffffffu, cgy = 0, cgz = 0, idx[8];
    float2 acc[8];
    bool dirty = false;
#pragma unroll 1
    for (int k = 0; k < RUN; ++k) {
        const uint32_t i = base + k;
        if (i >= n) break;
        const float2 d = to_f2(reinterpret_cast<const V*>(dy)[(size_t)i * N_LEVELS + level]);
        if (d.x == 0.f && d.y == 0.f) continue;
        const HashCell hc = hash_cell(lv, __ldg(x + 3 * (size_t)i), __ldg(x + 3 * (size_t)i + 1), __ldg(x + 3 * (size_t)i + 2));
        if (hc.gx != cgx || hc.gy != cgy || hc.gz != cgz) {
            if (dirty) {
                if constexpr (sizeof(T) == 2) red_add_corners(g, idx, acc);
                else {
#pragma unroll
                    for (int c = 0; c < 8; ++c) red_add(g + idx[c], acc[c].x, acc[c].y);
                }
            }
            cgx = hc.gx; cgy = hc.gy; cgz = hc.gz;
            hash_cell_indices(lv, cgx, cgy, cgz, idx);
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[c] = make_float2(0.f, 0.f);
            dirty = true;
        }
        float w[8];
        hash_cell_weights(hc, w);
#pragma unroll
        for (int c = 0; c < 8; ++c) { acc[c].x = fmaf(d.x, w[c], acc[c].x); acc[c].y = fmaf(d.y, w[c], acc[c].y); }
    }
    if (dirty) {
        if constexpr (sizeof(T) == 2) red_add_corners(g, idx, acc);
        else {
#pragma unroll
            for (int c = 0; c < 8; ++c) red_add(g + idx[c], acc[c].x, acc[c].y);
        }
    }
}

template <typename T>
__global__ void sh_kernel(uint32_t n, const float* __restrict__ dirs, T* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float o[16];
    sh4(dirs[3 * (size_t)i], dirs[3 * (size_t)i + 1], dirs[3 * (size_t)i + 2], o);
    if constexpr (sizeof(T) == 2) {
        uint32_t pk[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            __half2 h = __floats2half2_rn(o[2 * k], o[2 * k + 1]);
            pk[k] = *reinterpret_cast<uint32_t*>(&h);
        }
        uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * 16);
        dst[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        dst[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
    } else {
        float4* dst = reinterpret_cast<float4*>(out + (size_t)i * 16);
#pragma unroll
        for (int k = 0; k < 4; ++k) dst[k] = make_float4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
    }
}

}  // namespace

extern "C" {

int ngp_hash_offsets(double aabb_scale, int n_levels, int base_resolution, int log2_hashmap_size, uint32_t* offsets,
                     double* per_level_scale_out) {
    NGP_REQUIRE(n_levels >= 2 && n_levels <= 32 && offsets, "ngp_hash_offsets: bad arguments");
    // HE/grid_encode.py:19-36, python doubles
    const double pls = std::exp(std::log(2048.0 * aabb_scale / base_resolution) / (n_levels - 1));
    uint64_t offset = 0;
    for (int i = 0; i < n_levels; ++i) {
        const double scale = std::pow(2.0, i * std::log2(pls)) * base_resolution - 1.0;
        const uint64_t res = (uint64_t)std::ceil(scale) + 1;
        uint64_t params = res * res * res;
        params = ((params + 7) / 8) * 8;
        if (params > (1ull << log2_hashmap_size)) params = 1ull << log2_hashmap_size;
        offsets[i] = (uint32_t)offset;
        offset += params;
    }
    offsets[n_levels] = (uint32_t)offset;
    if (per_level_scale_out) *per_level_scale_out = pls;
    return 0;
}

int ngp_hash_level_table_primes(void* stream, const uint32_t* offsets_host, int n_levels, uint32_t base_resolution,
                                float log2_per_level_scale, void* levels_dev, uint32_t prime0, uint32_t prime1, uint32_t prime2) {
    NGP_REQUIRE(n_levels == N_LEVELS, "ngp_hash_level_table: the encoder is fixed at 16 levels (HE/hash_encoder.py:17-18)");
    cudaStream_t s = (cudaStream_t)stream;
    uint32_t* d_off = nullptr;
    NGP_CHECK_CUDA(cudaMallocAsync(&d_off, sizeof(uint32_t) * (n_levels + 1), s));   // init-time only
    NGP_CHECK_CUDA(cudaMemcpyAsync(d_off, offsets_host, sizeof(uint32_t) * (n_levels + 1), cudaMemcpyHostToDevice, s));
    level_table_kernel<<<1, 32, 0, s>>>(d_off, n_levels, base_resolution, log2_per_level_scale, (NgpLevel*)levels_dev, prime0, prime1, prime2);
    NGP_LAUNCH_CHECK();
    NGP_CHECK_CUDA(cudaFreeAsync(d_off, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    return 0;
}

int ngp_hash_level_table(void* stream, const uint32_t* offsets_host, int n_levels, uint32_t base_resolution,
                         float log2_per_level_scale, void* levels_dev) {
    // the configs' hash_func: p0 ^ p1 * 19349663 ^ p2 * 83492791 (projects/ngp/configs/ngp_base.py:66)
    return ngp_hash_level_table_primes(stream, offsets_host, n_levels, base_resolution, log2_per_level_scale, levels_dev, 1u, 19349663u, 83492791u);
}

int ngp_hash_fwd(void* stream, uint32_t n, const float* x, const void* grid, int dtype, const void* levels_dev, void* out) {
    if (n == 0) return 0;                                                  // HE/grid_encode.py:78-80
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t rb = (n + RUN_PTS_PER_BLOCK - 1) / RUN_PTS_PER_BLOCK;
    if (dtype == 1) hash_fwd_kernel<__half><<<rb, HASH_THREADS, 0, s>>>(n, x, (const __half*)grid, (const NgpLevel*)levels_dev, (__half*)out);
    else if (dtype == 0) hash_fwd_kernel<float><<<rb, HASH_THREADS, 0, s>>>(n, x, (const float*)grid, (const NgpLevel*)levels_dev, (float*)out);
    else NGP_REQUIRE(false, "ngp_hash_fwd: dtype must be 0 (f32) or 1 (f16)");
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_hash_bwd(void* stream, uint32_t n, const float* x, const void* dy, int dtype, const void* levels_dev, void* grid_grad,
                 uint64_t n_params) {
    NGP_REQUIRE(dtype == 0 || dtype == 1, "ngp_hash_bwd: dtype must be 0 (f32) or 1 (f16)");
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return 0;                                                  // HE/grid_encode.py:142-144 (returns before the memset)
    NGP_CHECK_CUDA(cudaMemsetAsync(grid_grad, 0, n_params * (dtype == 1 ? 2 : 4), s));   // :153
    const uint32_t rb = (n + RUN_PTS_PER_BLOCK - 1) / RUN_PTS_PER_BLOCK;
    if (dtype == 1) hash_bwd_kernel<__half><<<rb, HASH_THREADS, 0, s>>>(n, x, (const __half*)dy, (const NgpLevel*)levels_dev, (__half*)grid_grad);
    else hash_bwd_kernel<float><<<rb, HASH_THREADS, 0, s>>>(n, x, (const float*)dy, (const NgpLevel*)levels_dev, (float*)grid_grad);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_sh_fwd(void* stream, uint32_t n, const float* dirs, int dtype, void* out) {
    if (n == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == 1) sh_kernel<__half><<<(n + 127) / 128, 128, 0, s>>>(n, dirs, (__half*)out);
    else if (dtype == 0) sh_kernel<float><<<(n + 127) / 128, 128, 0, s>>>(n, dirs, (float*)out);
    else NGP_REQUIRE(false, "ngp_sh_fwd: dtype must be 0 (f32) or 1 (f16)");
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
