// Mip-NeRF cone casting and integrated positional encoding (utils/miputils.py:130-275 of the reference's contrib/mipnerf), shared by
// the fused network forward (mip_mlp.cu) and the fp32 encoder (mip_sampler.cu).  DESIGN.md section 11.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mip {
// A ray row: origin[3], direction[3] (unnormalised), viewdir[3], base radius, near, far.
constexpr uint32_t RAY_FLOATS = 12;
constexpr uint32_t IPE_DEGS = 8;                      // max_deg_point - min_deg_point: 48 encoding columns, the kernels' input width
constexpr uint32_t IPE_W = 6 * IPE_DEGS;
constexpr uint32_t VIEW_DEGS = 4;                     // deg_view: pos_enc(viewdir, 0, 4) is 27 wide
constexpr uint32_t MAX_SAMPLES = 128;                 // one warp a ray, four intervals a lane

// Coordinate `dim` of the mean and the diagonal covariance of the Gaussian of interval [t0, t1] of ray `ray`: the stable conical-frustum
// form (conical_frustum_to_gaussian, :159-190) or the cylinder (:193-212), lifted along the direction (lift_gaussian, diag, :138-148).
// integrate = 0 is disable_integration: covariance 0.
__device__ __forceinline__ void gaussian(const float* ray, float t0, float t1, uint32_t dim, bool cylinder, bool integrate, float& mean, float& var) {
    const float dx = ray[3], dy = ray[4], dz = ray[5], d = ray[3 + dim], r = ray[9];
    float t_mean, t_var, r_var;
    if (cylinder) {
        t_mean = (t0 + t1) / 2;
        r_var = r * r / 4;
        t_var = (t1 - t0) * (t1 - t0) / 12;
    } else {
        const float mu = (t0 + t1) / 2, hw = (t1 - t0) / 2, mu2 = mu * mu, hw2 = hw * hw, den = 3 * mu2 + hw2;
        t_mean = mu + (2 * mu * hw2) / den;
        t_var = hw2 / 3 - (4.f / 15.f) * ((hw2 * hw2 * (12 * mu2 - hw2)) / (den * den));
        r_var = r * r * (mu2 / 4 + (5.f / 12.f) * hw2 - (4.f / 15.f) * (hw2 * hw2) / den);
    }
    mean = d * t_mean + ray[dim];
    const float d_mag_sq = fmaxf(1e-10f, dx * dx + dy * dy + dz * dz);
    var = integrate ? t_var * (d * d) + r_var * (1.f - d * d / d_mag_sq) : 0.f;
}

// integrated_pos_enc (:242-275) of one coordinate: put(3k + dim, sin(y) e^(-var'/2)) and put(3 DEGS + 3k + dim, cos(y) e^(-var'/2)) with
// y = mean 2^(min_deg+k), var' = var 4^(min_deg+k), k < DEGS -- sin(y + pi/2) of the reference as cos(y), full-range sincosf (arguments
// reach several hundred radians at 8 degrees, ~1e5 at 16).
template <uint32_t DEGS = IPE_DEGS, class Put>
__device__ __forceinline__ void ipe(float mean, float var, uint32_t dim, int min_deg, Put put) {
#pragma unroll
    for (uint32_t k = 0; k < DEGS; ++k) {
        const float s = ldexpf(1.f, min_deg + (int)k);
        const float e = expf(-0.5f * (var * (s * s)));
        float sn, cs;
        sincosf(mean * s, &sn, &cs);
        put(3 * k + dim, sn * e);
        put(3 * DEGS + 3 * k + dim, cs * e);
    }
}

// Blender camera direction (dataset/nerf_datasets.py:193-235, dataset/nerf.py:265-276): camera_dirs = [(x - W/2 + 0.5) / f,
// -(y - H/2 + 0.5) / f, -1], direction = camera_dirs @ R^T, in fp32 in numpy's order (callers are built with -fmad=false).
__device__ __forceinline__ void cam_dir(const float* c2w, float x, float y, uint32_t W, uint32_t H, float focal, float d[3]) {
    const float cx = (x - W * 0.5f + 0.5f) / focal, cy = -((y - H * 0.5f + 0.5f) / focal), cz = -1.f;
#pragma unroll
    for (int j = 0; j < 3; ++j) d[j] = cx * c2w[4 * j] + cy * c2w[4 * j + 1] + cz * c2w[4 * j + 2];
}
}  // namespace mip
