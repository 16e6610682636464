// oracle/_ref build (SURVEY.md F1): the reference's own CUDA kernels compiled UNMODIFIED for sm_90a, each header in
// its own namespace, behind extern "C" launchers that replicate the reference's launch shapes (SURVEY.md 2b).
// TEST / BENCH INFRASTRUCTURE: the GPU comparator ("the kernel to beat") and the bit-exactness anchor for sample
// indices (SURVEY.md H4).  Never linked into libngp_b200.so.  Compile with -DREF_CONST_DT=1 (lego) or 0 (fox).
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <atomic>
#include <limits>
#include <stdexcept>
#include <vector>
#include <cassert>
#include <Eigen/Core>
#include <Eigen/Dense>
#include "pcg32.h"

// ---- generated constants prelude, as DGS/density_grid_sampler.py:96-116 emits it ----------
inline constexpr __device__ __host__ uint32_t NERF_GRIDSIZE() { return 128; }
inline constexpr __device__ __host__ float NERF_RENDERING_NEAR_DISTANCE() { return 0.05f; }
inline constexpr __device__ __host__ uint32_t NERF_STEPS() { return 1024; }
inline constexpr __device__ __host__ uint32_t NERF_CASCADES() { return 5; }
inline __device__ float NERF_MIN_OPTICAL_THICKNESS() { return 0.01f; }
inline constexpr __device__ __host__ float SQRT3() { return 1.73205080757f; }
inline constexpr __device__ __host__ float STEPSIZE() { return (SQRT3() / NERF_STEPS()); }
inline constexpr __device__ __host__ float MIN_CONE_STEPSIZE() { return STEPSIZE(); }
inline constexpr __device__ __host__ float MAX_CONE_STEPSIZE() { return STEPSIZE() * (1 << (NERF_CASCADES() - 1)) * NERF_STEPS() / NERF_GRIDSIZE(); }
#if REF_CONST_DT
inline __device__ __host__ float calc_dt(float t, float cone_angle) { return MIN_CONE_STEPSIZE() * 0.5; }
#define SUFFIX(name) name##_constdt
#else
inline __device__ __host__ float clamp_(float val, float lower, float upper) { return val < lower ? lower : (upper < val ? upper : val); }
inline __device__ __host__ float calc_dt(float t, float cone_angle) { return clamp_(t * cone_angle, MIN_CONE_STEPSIZE(), MAX_CONE_STEPSIZE()); }
#define SUFFIX(name) name##_cone
#endif

#define get_index(p0, p1, p2) p0 ^ p1 * 19349663 ^ p2 * 83492791
namespace g_hash {
#include "HashEncode.h"
}
namespace g_march {
#include "ray_sampler.h"
}
namespace g_compact {
#include "compacted_coord.h"
}
namespace g_rgb {
#include "calc_rgb.h"
}

static pcg32 make_rng(uint64_t state, uint64_t inc) {
    pcg32 r;
    r.state = state;
    r.inc = inc;
    return r;
}

extern "C" {

// HE/grid_encode.py:66-129 : extract_position (64,3) -> kernel_grid 512 x (.,16) -> transpose (16,8)
int SUFFIX(refgpu_hash_fwd_f16)(uint32_t n, const float* x, const void* grid, const uint32_t* offsets, float log2_pls, float* pos_soa,
                                void* enc_soa, void* out) {
    using namespace g_hash;
    const dim3 threads = {64, 3, 1};
    extract_position<float, 3><<<div_round_up(n, 64u), threads>>>(n, PitchedPtr<const float>(x, 3), pos_soa);
    const dim3 blocks_hashgrid = {div_round_up(n, 512u), 16, 1};
    kernel_grid<__half, 3, 2><<<blocks_hashgrid, 512>>>(n, 32, offsets, 16, log2_pls, 0.0f, 1000.0f, 1, 0, (const __half*)grid, pos_soa,
                                                       (vector_t<__half, 2>*)enc_soa, nullptr);
    const dim3 threads_transpose = {16, 8, 1};
    transpose_encoded_position<vector_t<__half, 2>><<<div_round_up(n, 8u), threads_transpose>>>(
        n, (const vector_t<__half, 2>*)enc_soa, PitchedPtr<vector_t<__half, 2>>((vector_t<__half, 2>*)out, 16));
    return (int)cudaGetLastError();
}
int SUFFIX(refgpu_hash_fwd_f32)(uint32_t n, const float* x, const float* grid, const uint32_t* offsets, float log2_pls, float* pos_soa,
                                float* enc_soa, float* out) {
    using namespace g_hash;
    const dim3 threads = {64, 3, 1};
    extract_position<float, 3><<<div_round_up(n, 64u), threads>>>(n, PitchedPtr<const float>(x, 3), pos_soa);
    const dim3 blocks_hashgrid = {div_round_up(n, 512u), 16, 1};
    kernel_grid<float, 3, 2><<<blocks_hashgrid, 512>>>(n, 32, offsets, 16, log2_pls, 0.0f, 1000.0f, 1, 0, grid, pos_soa,
                                                      (vector_t<float, 2>*)enc_soa, nullptr);
    const dim3 threads_transpose = {16, 8, 1};
    transpose_encoded_position<vector_t<float, 2>><<<div_round_up(n, 8u), threads_transpose>>>(
        n, (const vector_t<float, 2>*)enc_soa, PitchedPtr<vector_t<float, 2>>((vector_t<float, 2>*)out, 16));
    return (int)cudaGetLastError();
}
// HE/grid_encode.py:131-190 : memset + transpose_gradients + kernel_grid_backward 256 x (.,16)
int SUFFIX(refgpu_hash_bwd_f16)(uint32_t n, const float* pos_soa, const void* dy, const uint32_t* offsets, float log2_pls, void* dy_soa,
                                void* grid_grad, uint64_t n_params) {
    using namespace g_hash;
    cudaMemsetAsync(grid_grad, 0, n_params * 2);
    const dim3 threads_transpose = {16, 8, 1};
    transpose_gradients<vector_t<__half, 2>><<<div_round_up(n, 8u), threads_transpose>>>(
        n, (vector_t<__half, 2>*)dy_soa, PitchedPtr<const vector_t<__half, 2>>((const vector_t<__half, 2>*)dy, 16));
    const dim3 blocks_hashgrid = {div_round_up(n, 256u), 16, 1};
    kernel_grid_backward<__half, __half, 3, 2, 2><<<blocks_hashgrid, 256>>>(n, 32, offsets, 16, log2_pls, 1000.0f, false, 1, 0,
                                                                            (__half*)grid_grad, pos_soa, (const vector_t<__half, 2>*)dy_soa);
    return (int)cudaGetLastError();
}

// DGS/ray_sampler.py:20-72 (including its 117 MB-style memset of the whole output buffer)
int SUFFIX(refgpu_march)(uint32_t n_rays, float aabb_min, float aabb_max, uint32_t max_samples, const float* rays_o, const float* rays_d,
                         const uint8_t* bitfield, float cone_angle, const float* metadata, const uint32_t* imgs_index, uint32_t* counters,
                         uint32_t* ray_indices, uint32_t* numsteps, float* coords_out, const float* xforms, float near_distance,
                         uint64_t rng_state, uint64_t rng_inc, int do_memset) {
    using namespace g_march;
    BoundingBox aabb(Eigen::Vector3f::Constant(aabb_min), Eigen::Vector3f::Constant(aabb_max));
    cudaMemsetAsync(counters, 0, 8);
    if (do_memset) cudaMemsetAsync(coords_out, 0, (size_t)max_samples * 28);
    linear_kernel(rays_sampler, 0, 0, n_rays, aabb, max_samples, (Vector3f*)rays_o, (Vector3f*)rays_d, (uint8_t*)bitfield, cone_angle,
                  (TrainingImageMetadata*)metadata, (uint32_t*)imgs_index, counters, counters + 1, ray_indices, numsteps,
                  PitchedPtr<NerfCoordinate>((NerfCoordinate*)coords_out, 1, 0, 0), (Eigen::Matrix<float, 3, 4>*)xforms, near_distance,
                  make_rng(rng_state, rng_inc));
    return (int)cudaGetLastError();
}

// DGS/compacted_coord.py:28-70
int SUFFIX(refgpu_compact_f16)(uint32_t n_rays, uint32_t max_compacted, const void* net_out, const float* coords_in, float* coords_out,
                               const uint32_t* numsteps_in, uint32_t* numsteps_counter, uint32_t* numsteps_out, uint32_t* rays_counter) {
    using namespace g_compact;
    BoundingBox aabb(Eigen::Vector3f::Constant(0.f), Eigen::Vector3f::Constant(1.f));
    cudaMemsetAsync(numsteps_counter, 0, 4);
    cudaMemsetAsync(rays_counter, 0, 4);
    cudaMemsetAsync(coords_out, 0, (size_t)max_compacted * 28);
    linear_kernel(compacted_coord<__half>, 0, 0, n_rays, aabb, max_compacted, 4, Array4f(1, 1, 1, 1), (const __half*)net_out, ENerfActivation(2),
                  ENerfActivation(3), (const NerfCoordinate*)coords_in, (NerfCoordinate*)coords_out, numsteps_in, numsteps_counter, numsteps_out,
                  rays_counter);
    return (int)cudaGetLastError();
}

// DGS/calc_rgb.py:31-108
int SUFFIX(refgpu_rgb_fwd_f16)(uint32_t n_rays, const void* net_out, const float* coords, const uint32_t* numsteps_in, float* rgb_out,
                               const uint32_t* numsteps_compacted, const float* bg) {
    using namespace g_rgb;
    BoundingBox aabb(Eigen::Vector3f::Constant(0.f), Eigen::Vector3f::Constant(1.f));
    linear_kernel(compute_rgbs<__half>, 0, 0, n_rays, aabb, 4, (const __half*)net_out, ENerfActivation(2), ENerfActivation(3),
                  PitchedPtr<NerfCoordinate>((NerfCoordinate*)coords, 1, 0, 0), (uint32_t*)numsteps_in, (Array3f*)rgb_out,
                  (uint32_t*)numsteps_compacted, (const Array3f*)bg, (int)NERF_CASCADES(), MIN_CONE_STEPSIZE());
    return (int)cudaGetLastError();
}
int SUFFIX(refgpu_rgb_bwd_f16)(uint32_t n_rays, uint32_t n_elements, void* dloss_doutput, const void* net_out, const uint32_t* numsteps_compacted,
                               const float* coords, const float* loss_grad, const float* rgb_ray, const float* density_grid_mean) {
    using namespace g_rgb;
    BoundingBox aabb(Eigen::Vector3f::Constant(0.f), Eigen::Vector3f::Constant(1.f));
    cudaMemsetAsync(dloss_doutput, 0, (size_t)n_elements * 8);
    linear_kernel(compute_rgbs_grad<__half>, 0, 0, n_rays, aabb, 4, (__half*)dloss_doutput, (const __half*)net_out, (uint32_t*)numsteps_compacted,
                  PitchedPtr<NerfCoordinate>((NerfCoordinate*)coords, 1, 0, 0), ENerfActivation(2), ENerfActivation(3), (Array3f*)loss_grad,
                  (Array3f*)rgb_ray, (float*)density_grid_mean, (int)NERF_CASCADES(), MIN_CONE_STEPSIZE());
    return (int)cudaGetLastError();
}
}
