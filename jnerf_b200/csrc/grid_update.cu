// R10: occupancy-grid maintenance (DGS/density_grid_sampler.py:204-264): mark_untrained, sample generation,
// max-splat, decayed max, mean, bitfield and max-pool.  Restated from the five small reference headers
// (mark_untrained_density_grid.h, generate_grid_samples_nerf_nonuniform.h, splat_grid_samples_nerf_max_nearest_neighbor.h,
// ema_grid_samples_nerf.h, update_bitfield.h).  Compiled with -fmad=false; explicit order of operations follows the
// oracle.  The grid mean uses a fixed-order two-stage reduction (the reference's atomicAdd order is nondeterministic):
// data-parallel replicas must derive bit-identical bitfields from bit-identical grids.
#include "ngp_common.cuh"

namespace {

__global__ void mark_untrained_kernel(uint32_t n_elements, float* __restrict__ grid, uint32_t n_images, const float* __restrict__ focal,
                                      const float* __restrict__ xforms, float half_resx, float half_resy) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_elements) return;
    const uint32_t level = i / NERF_GRID_N, pos_idx = i % NERF_GRID_N;
    const uint32_t x = morton3D_invert(pos_idx >> 0), y = morton3D_invert(pos_idx >> 1), z = morton3D_invert(pos_idx >> 2);
    const float sc = scalbnf(1.0f, (int)level);
    const float p[3] = {(((float)x + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f, (((float)y + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f,
                        (((float)z + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f};
    const float voxel_radius = 0.5f * 1.73205080757f * sc / NERF_GRIDSIZE;
    int count = 0;
    for (uint32_t j = 0; j < n_images; ++j) {
        const float* m = xforms + 12 * j;   // column-major 3x4 (dataset/dataset.py:164-165)
        const float pl[3] = {p[0] - __ldg(m + 9), p[1] - __ldg(m + 10), p[2] - __ldg(m + 11)};
        const float cx = pl[0] * __ldg(m + 0) + (pl[1] * __ldg(m + 1) + pl[2] * __ldg(m + 2));
        const float cy = pl[0] * __ldg(m + 3) + (pl[1] * __ldg(m + 4) + pl[2] * __ldg(m + 5));
        const float cz = pl[0] * __ldg(m + 6) + (pl[1] * __ldg(m + 7) + pl[2] * __ldg(m + 8));
        if (cz > 0.f) {
            if (fabsf(cx) - voxel_radius < cz / __ldg(focal + 2 * j) * half_resx && fabsf(cy) - voxel_radius < cz / __ldg(focal + 2 * j + 1) * half_resy) {
                count++;
                break;
            }
        }
    }
    if ((grid[i] < 0) != (count <= 0)) grid[i] = (count > 0) ? 0.f : -1.f;
}

// mark_untrained_kernel for captures whose frames carry their own cameras: a cell is seen by image j when its bounding sphere reaches
// into the image's frustum, x_lo < c_x / c_z < x_hi and y_lo < c_y / c_z < y_hi, with the image's normalised extents (x_lo, x_hi,
// y_lo, y_hi) = extents[j] computed on the host (plugin/dataset.py: frame_extent) from its size, principal point, focal lengths and
// lens.  The symmetric |c_x| < c_z (W/2) / f test above holds only for a centred principal point.
__global__ void mark_untrained_cams_kernel(uint32_t n_elements, float* __restrict__ grid, uint32_t n_images, const float4* __restrict__ extents,
                                           const float* __restrict__ xforms) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_elements) return;
    const uint32_t level = i / NERF_GRID_N, pos_idx = i % NERF_GRID_N;
    const uint32_t x = morton3D_invert(pos_idx >> 0), y = morton3D_invert(pos_idx >> 1), z = morton3D_invert(pos_idx >> 2);
    const float sc = scalbnf(1.0f, (int)level);
    const float p[3] = {(((float)x + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f, (((float)y + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f,
                        (((float)z + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f};
    const float voxel_radius = 0.5f * 1.73205080757f * sc / NERF_GRIDSIZE;
    bool seen = false;
    for (uint32_t j = 0; j < n_images && !seen; ++j) {
        const float* m = xforms + 12 * j;
        const float pl[3] = {p[0] - __ldg(m + 9), p[1] - __ldg(m + 10), p[2] - __ldg(m + 11)};
        const float cx = pl[0] * __ldg(m + 0) + (pl[1] * __ldg(m + 1) + pl[2] * __ldg(m + 2));
        const float cy = pl[0] * __ldg(m + 3) + (pl[1] * __ldg(m + 4) + pl[2] * __ldg(m + 5));
        const float cz = pl[0] * __ldg(m + 6) + (pl[1] * __ldg(m + 7) + pl[2] * __ldg(m + 8));
        if (cz > 0.f) {
            const float4 e = __ldg(extents + j);
            seen = cx + voxel_radius > cz * e.x && cx - voxel_radius < cz * e.y && cy + voxel_radius > cz * e.z && cy - voxel_radius < cz * e.w;
        }
    }
    if ((grid[i] < 0) != !seen) grid[i] = seen ? 0.f : -1.f;
}

__global__ void generate_samples_kernel(uint32_t n_elements, uint64_t rng_state, uint64_t rng_inc, const uint32_t* __restrict__ step_p,
                                        float lo, float hi, const float* __restrict__ grid_in, float* __restrict__ positions,
                                        uint32_t* __restrict__ indices, uint32_t n_cascades, float thresh) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_elements) return;
    Pcg32 rng{rng_state, rng_inc};
    rng.advance((int64_t)(uint32_t)(i * 4u));
    const uint32_t level = (uint32_t)(rng.next_float() * n_cascades) % n_cascades;
    const uint32_t step = *step_p;
    uint32_t idx = 0;
    for (uint32_t j = 0; j < 10; ++j) {
        idx = ((i + step * n_elements) * 56924617u + j * 19349663u + 96925573u) % NERF_GRID_N;
        idx += level * NERF_GRID_N;
        if (grid_in[idx] > thresh) break;
    }
    const uint32_t pos_idx = idx % NERF_GRID_N;
    const uint32_t x = morton3D_invert(pos_idx >> 0), y = morton3D_invert(pos_idx >> 1), z = morton3D_invert(pos_idx >> 2);
    const float r0 = rng.next_float(), r1 = rng.next_float(), r2 = rng.next_float();
    const float sc = scalbnf(1.0f, (int)level), diag = hi - lo;
    const float p[3] = {(((float)x + r0) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f, (((float)y + r1) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f,
                        (((float)z + r2) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f};
    positions[3 * (size_t)i] = (p[0] - lo) / diag;
    positions[3 * (size_t)i + 1] = (p[1] - lo) / diag;
    positions[3 * (size_t)i + 2] = (p[2] - lo) / diag;
    indices[i] = idx;
}

template <typename T>
__global__ void splat_kernel(uint32_t n, const uint32_t* __restrict__ indices, const T* __restrict__ mlp_out, float* __restrict__ grid_tmp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float mlp = __expf((float)mlp_out[i]);                       // network_to_density, Exponential
    const float thick = mlp * (1.73205080757f / 1024.0f);              // scalbnf(MIN_CONE_STEPSIZE(), 0)
    atomicMax(reinterpret_cast<uint32_t*>(grid_tmp) + indices[i], __float_as_uint(thick));
}

__global__ void ema_kernel(uint32_t n, float decay, float* __restrict__ grid, const float* __restrict__ grid_tmp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float prev = grid[i];
    grid[i] = (prev < 0.f) ? prev : fmaxf(prev * decay, grid_tmp[i]);
}

constexpr int MEAN_BLOCKS = 256;
__global__ void __launch_bounds__(256) mean_partial_kernel(const float* __restrict__ grid, float* __restrict__ partial) {
    __shared__ float s[256];
    float acc = 0.f;
    const uint32_t per_block = NERF_GRID_N / MEAN_BLOCKS;   // 8192
    const float* g = grid + (size_t)blockIdx.x * per_block;
    for (uint32_t k = threadIdx.x; k < per_block; k += 256) acc += fmaxf(g[k], 0.f) / NERF_GRID_N;
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) s[threadIdx.x] += s[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}
__global__ void __launch_bounds__(256) mean_final_kernel(const float* __restrict__ partial, float* __restrict__ mean) {
    __shared__ float s[256];
    s[threadIdx.x] = partial[threadIdx.x];
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) s[threadIdx.x] += s[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) *mean = s[0];
}

__global__ void grid_to_bitfield_kernel(uint32_t n, const float* __restrict__ grid, uint8_t* __restrict__ bits, const float* __restrict__ mean) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float m = *mean;
    const float thresh = 0.01f < m ? 0.01f : m;
    const float4 a = reinterpret_cast<const float4*>(grid)[2 * (size_t)i], b = reinterpret_cast<const float4*>(grid)[2 * (size_t)i + 1];
    uint8_t v = 0;
    v |= a.x > thresh ? 1 : 0; v |= a.y > thresh ? 2 : 0; v |= a.z > thresh ? 4 : 0; v |= a.w > thresh ? 8 : 0;
    v |= b.x > thresh ? 16 : 0; v |= b.y > thresh ? 32 : 0; v |= b.z > thresh ? 64 : 0; v |= b.w > thresh ? 128 : 0;
    bits[i] = v;
}
__global__ void bitfield_max_pool_kernel(uint32_t n, const uint8_t* __restrict__ prev, uint8_t* __restrict__ next) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint2 p = reinterpret_cast<const uint2*>(prev)[i];
    uint8_t bits = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        bits |= ((p.x >> (8 * j)) & 0xFF) ? (uint8_t)(1 << j) : 0;
        bits |= ((p.y >> (8 * j)) & 0xFF) ? (uint8_t)(1 << (4 + j)) : 0;
    }
    const uint32_t x = morton3D_invert(i >> 0) + NERF_GRIDSIZE / 8, y = morton3D_invert(i >> 1) + NERF_GRIDSIZE / 8,
                   z = morton3D_invert(i >> 2) + NERF_GRIDSIZE / 8;
    next[morton3D(x, y, z)] |= bits;
}

float* g_mean_partial = nullptr;

}  // namespace

extern "C" {

int ngp_grid_mark_untrained(void* stream, uint32_t n_elements, float* grid, uint32_t n_images, const float* focal_lengths, const float* xforms,
                            int res_x, int res_y) {
    if (n_elements == 0) return 0;
    mark_untrained_kernel<<<(n_elements + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_elements, grid, n_images, focal_lengths, xforms,
                                                                                     res_x * 0.5f, res_y * 0.5f);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_grid_mark_untrained_cams(void* stream, uint32_t n_elements, float* grid, uint32_t n_images, const float* extents, const float* xforms) {
    if (n_elements == 0) return 0;
    NGP_REQUIRE(extents != nullptr && (reinterpret_cast<uintptr_t>(extents) & 15) == 0,
                "ngp_grid_mark_untrained_cams: extents must be a 16-byte aligned (n_images, 4) float array");
    mark_untrained_cams_kernel<<<(n_elements + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_elements, grid, n_images,
                                                                                          reinterpret_cast<const float4*>(extents), xforms);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_grid_generate_samples(void* stream, uint32_t n_elements, uint64_t rng_state, uint64_t rng_inc, const uint32_t* step_dev, float aabb_lo,
                              float aabb_hi, const float* grid_in, float* positions_out, uint32_t* indices_out, uint32_t n_cascades, float thresh) {
    if (n_elements == 0) return 0;   // linear_kernel returns for n_elements <= 0 (density_grid_sampler_header.h:26-33)
    generate_samples_kernel<<<(n_elements + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_elements, rng_state, rng_inc, step_dev, aabb_lo, aabb_hi,
                                                                                       grid_in, positions_out, indices_out, n_cascades, thresh);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_grid_splat(void* stream, uint32_t n, const uint32_t* indices, const void* mlp_out, int dtype, float* grid_tmp) {
    if (n == 0) return 0;
    if (dtype == 1) splat_kernel<__half><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, indices, (const __half*)mlp_out, grid_tmp);
    else if (dtype == 0) splat_kernel<float><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, indices, (const float*)mlp_out, grid_tmp);
    else NGP_REQUIRE(false, "ngp_grid_splat: bad dtype");
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_grid_ema(void* stream, uint32_t n_elements, float decay, float* grid, const float* grid_tmp) {
    if (n_elements == 0) return 0;
    ema_kernel<<<(n_elements + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_elements, decay, grid, grid_tmp);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_grid_update_bitfield(void* stream, const float* grid, float* mean_out, uint8_t* bitfield, uint32_t cascades) {
    NGP_REQUIRE(cascades >= 1 && cascades <= 8, "ngp_grid_update_bitfield: cascades out of range");
    NGP_REQUIRE(((size_t)grid) % 16 == 0, "Can only reduce_sum on 16-byte aligned memory.");   // update_bitfield.h:14-17
    cudaStream_t s = (cudaStream_t)stream;
    if (!g_mean_partial) NGP_CHECK_CUDA(cudaMalloc(&g_mean_partial, MEAN_BLOCKS * sizeof(float)));   // 1 KB scratch, once
    mean_partial_kernel<<<MEAN_BLOCKS, 256, 0, s>>>(grid, g_mean_partial);
    mean_final_kernel<<<1, 256, 0, s>>>(g_mean_partial, mean_out);
    const uint32_t n = NERF_GRID_N / 8 * cascades;
    grid_to_bitfield_kernel<<<(n + 127) / 128, 128, 0, s>>>(n, grid, bitfield, mean_out);
    for (uint32_t level = 1; level < cascades; ++level) {
        bitfield_max_pool_kernel<<<(NERF_GRID_N / 64 + 127) / 128, 128, 0, s>>>(NERF_GRID_N / 64, bitfield + (size_t)NERF_GRID_N * (level - 1) / 8,
                                                                                bitfield + (size_t)NERF_GRID_N * level / 8);
    }
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
