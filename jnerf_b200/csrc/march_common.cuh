// Ray-march and sample helpers shared by the march of sampler.cu and the wavefront renderer of render.cu: the step rule of
// DGS/op_header/ray_sampler.h:4-114 and ray_sampler_header.h (calc_dt, mip level, occupancy test, voxel skip, slab test, jitter) and
// the per-sample terms of the composite (calc_rgb.h).  One definition, so that both files take the same steps bit for bit.  Every file
// that includes this is compiled with -fmad=false: the multiply-adds the reference's GPU build contracts are written as __fmaf_rn.
#pragma once
#include "ngp_common.cuh"
#include <cfloat>

namespace {

struct MarchCfg {
    uint32_t cascades;
    int const_dt;
    float min_cone, max_cone;
};
__host__ __device__ inline MarchCfg make_cfg(uint32_t cascades, int const_dt) {
    MarchCfg c;
    c.cascades = cascades;
    c.const_dt = const_dt;
    c.min_cone = 1.73205080757f / 1024.0f;                                   // STEPSIZE(), density_grid_sampler.py:102-104
    c.max_cone = c.min_cone * (float)(1u << (cascades - 1)) * 1024.0f / 128.0f;  // :105 (all factors are powers of two)
    return c;
}
__device__ __forceinline__ float calc_dt(const MarchCfg& c, float t, float cone) {
    if (c.const_dt) return c.min_cone * 0.5f;                                // density_grid_sampler.py:107-110
    // :112-115 clamp(t * cone, min, max), branch-free (identical for every non-NaN t; a NaN t ends the ray at its next bounds test anyway)
    return fminf(fmaxf(t * cone, c.min_cone), c.max_cone);
}
// The exponent frexpf(x, &e) returns, for x >= 0 as the callers below use it: exponent field - 126 for every normal float, 0 for
// x = 0; a denormal x (true exponent < -125) reads -126 here, which the callers clamp to the same result.
__device__ __forceinline__ int frexp_exponent(float x) { return x == 0.f ? 0 : (int)((__float_as_uint(x) >> 23) & 0xffu) - 126; }
__device__ __forceinline__ int mip_from_pos(const MarchCfg& c, float px, float py, float pz) {
    const float m = fmaxf(fmaxf(fabsf(px - 0.5f), fabsf(py - 0.5f)), fabsf(pz - 0.5f));
    return min((int)c.cascades - 1, max(0, frexp_exponent(m) + 1));           // ray_sampler_header.h:60-66
}
__device__ __forceinline__ int mip_from_dt(const MarchCfg& c, float dt, float px, float py, float pz) {
    const int mip = mip_from_pos(c, px, py, pz);
    dt *= 2 * NERF_GRIDSIZE;
    if (dt < 1.f) return mip;
    return min((int)c.cascades - 1, max(frexp_exponent(dt), mip));            // :68-77
}
__device__ __forceinline__ uint32_t grid_idx_at(float px, float py, float pz, uint32_t mip) {
    const float s = __uint_as_float((127u - mip) << 23);                     // scalbnf(1, -mip), :755-770
    float q[3] = {px, py, pz};
    int ix[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float v = q[d] - 0.5f;
        v *= s;
        v += 0.5f;
        const int i = (int)(v * NERF_GRIDSIZE);
        ix[d] = min(max(i, 0), (int)NERF_GRIDSIZE - 1);
    }
    return morton3D(ix[0], ix[1], ix[2]);
}
__device__ __forceinline__ bool occupied_at(float px, float py, float pz, const uint8_t* __restrict__ bits, uint32_t mip) {
    const uint32_t idx = grid_idx_at(px, py, pz, mip);
    return __ldg(bits + idx / 8 + (NERF_GRID_N / 8) * mip) & (1 << (idx % 8));   // :772-776
}
__device__ __forceinline__ float sgn(float x) { return copysignf(1.0f, x); }
// t + distance_to_next_voxel (ray_sampler_header.h:728-737, 747): where the empty-space skip of advance_to_next_voxel stops stepping
__device__ __forceinline__ float next_voxel_target(float t, const float p_[3], const float d[3], const float id[3], uint32_t res) {
    const float r = (float)res;
    const float p[3] = {r * p_[0], r * p_[1], r * p_[2]};
    const float tx = (floorf(p[0] + 0.5f + 0.5f * sgn(d[0])) - p[0]) * id[0];
    const float ty = (floorf(p[1] + 0.5f + 0.5f * sgn(d[1])) - p[1]) * id[1];
    const float tz = (floorf(p[2] + 0.5f + 0.5f * sgn(d[2])) - p[2]) * id[2];
    const float tt = fminf(fminf(tx, ty), tz);
    return t + fmaxf(tt / r, 0.0f);
}
// :739-753 as the reference writes it: unbounded (a ray whose t no longer grows, t + dt == t, would never reach the target).  The
// marches here bound the steps instead, see MARCH_STEP_GUARD.
__device__ __forceinline__ float advance_to_next_voxel(const MarchCfg& c, float t, float cone, const float p_[3], const float d[3],
                                                       const float id[3], uint32_t res) {
    const float t_target = next_voxel_target(t, p_, d, id, res);
    do { t += calc_dt(c, t, cone); } while (t < t_target);
    return t;
}
// Steps of the t sequence t_{k+1} = t_k + calc_dt(t_k) a ray may take, occupied or skipped: the samples of a ray are those with k below
// this bound.  Without it a ray whose t stops growing (t + dt == t: far from its origin, e.g. an origin ~16 k units from the box with
// const_dt, or a direction with all components below ~1e-6) or whose skip target is infinite (zero direction) would march for ever,
// where the reference hangs.  A ray of unit direction inside the box takes at most a few thousand steps.
constexpr uint32_t MARCH_STEP_GUARD = 1u << 20;
__device__ __forceinline__ bool contains(float lo, float hi, const float p[3]) {
    return p[0] >= lo && p[0] <= hi && p[1] >= lo && p[1] <= hi && p[2] >= lo && p[2] <= hi;
}
__device__ __forceinline__ float ray_tmin(float lo, float hi, const float o[3], const float d[3]) {
    float tmin = (lo - o[0]) / d[0], tmax = (hi - o[0]) / d[0], t;           // :408-465
    if (tmin > tmax) { t = tmin; tmin = tmax; tmax = t; }
    float tymin = (lo - o[1]) / d[1], tymax = (hi - o[1]) / d[1];
    if (tymin > tymax) { t = tymin; tymin = tymax; tymax = t; }
    if (tmin > tymax || tymin > tmax) return FLT_MAX;
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    float tzmin = (lo - o[2]) / d[2], tzmax = (hi - o[2]) / d[2];
    if (tzmin > tzmax) { t = tzmin; tzmin = tzmax; tzmax = t; }
    if (tmin > tzmax || tzmin > tmax) return FLT_MAX;
    if (tzmin > tmin) tmin = tzmin;
    return tmin;
}

struct RayState {
    float o[3], d[3], id[3], startt;
};
// `ray_offset` = index of ray 0 in the global ray batch (data-parallel shards draw the jitter of the global ray id)
struct MarchRng { uint64_t state, inc; uint32_t ray_offset; };
__device__ __forceinline__ RayState ray_setup(uint32_t i, const float* __restrict__ rays_o, const float* __restrict__ rays_d, float lo,
                                              float hi, float near_distance, float cone, const MarchCfg& c, const MarchRng& mr) {
    RayState r;
#pragma unroll
    for (int k = 0; k < 3; ++k) { r.o[k] = rays_o[3 * (size_t)i + k]; r.d[k] = rays_d[3 * (size_t)i + k]; r.id[k] = 1.0f / r.d[k]; }
    Pcg32 rng{mr.state, mr.inc};
    rng.advance((int64_t)(uint32_t)((i + mr.ray_offset) * 8u));               // ray_sampler.h:30, N_MAX_RANDOM_SAMPLES_PER_RAY = 8
    float tmin = fmaxf(ray_tmin(lo, hi, r.o, r.d), near_distance);           // :41-44
    r.startt = __fmaf_rn(calc_dt(c, tmin, cone), rng.next_float(), tmin);    // :48
    return r;
}

struct Sample {
    float rgb[3], alpha, dt, sigma_raw;
};
// 1 / (1 + e^-x) on the special-function unit: ex2.approx and rcp (2 ulp each) instead of expf + an IEEE division with its
// slow-path call -- three of these per sample were most of the instructions of the per-ray loop.  |error| < 1e-6 on a colour in
// [0, 1]; the radiance bar against the oracle is 1e-3 (tests/test_gpu_parity_e2e.py asserts 2e-4).
__device__ __forceinline__ float logistic_sfu(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ Sample make_sample(const float4& o, float dt_warped, uint32_t cascades) {   // network_to_rgb (Logistic), network_to_density (Exponential)
    Sample s;
    s.rgb[0] = logistic_sfu(o.x); s.rgb[1] = logistic_sfu(o.y); s.rgb[2] = logistic_sfu(o.z);
    s.dt = nerf_unwarp_dt(dt_warped, cascades);
    const float density = __expf(o.w);
    s.alpha = 1.f - __expf(-density * s.dt);
    s.sigma_raw = o.w;
    return s;
}

}  // namespace
