// Device helpers of the Plenoxels (svox2) kernels in svox.cu: the sparse grid behind a link table, the ray set-up of the reference's
// contrib/plenoxel render_util.cuh (world -> grid transform, box clipping, step in world units), trilinear interpolation through links
// (a link < 0 reads 0), the degree-2 SH basis, and the signed 64-bit fixed-point gradient sums.  DESIGN.md section 12.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace svox {
constexpr int BASIS = 9;                   // SH degree 2
constexpr int DATA_DIM = 3 * BASIS;        // sh_data columns: channel-major (r: 0-8, g: 9-17, b: 18-26)
constexpr uint32_t FULL = 0xffffffffu;
// Fixed point: one unit is 2^-48 of a gradient.  A single term must stay below 2^14 so that it converts without saturating; the
// sums are checked for signed overflow (|sum| < 2^15).  DESIGN.md section 12 derives both bounds.
constexpr float FX_SCALE = 281474976710656.f;             // 2^48
constexpr float FX_UNIT = 3.5527136788005009e-15f;        // 2^-48
constexpr float FX_MAX_TERM = 16384.f;                    // 2^14

// The grid in the coordinates of the kernels: links (size[0], size[1], size[2]) row-major, density (capacity), sh (capacity, 27).
// offset / scaling map world to grid coordinates, p_grid = p_world * scaling + offset (_offset * reso - 0.5 and _scaling * reso).
struct Grid {
    const int32_t* links;
    const float* density;
    const float* sh;
    int size[3];
    float offset[3], scaling[3];
};
// RenderOptions (svox2_utils.py:338-372) as the reference runs them: step 0.5, sigma_thresh 1e-10, stop_thresh 1e-7, background 1.
struct Opt {
    float step_size, sigma_thresh, stop_thresh, background;
};
struct Ray {
    float o[3], d[3];
    float tmin, tmax, world_step;
};

__device__ __forceinline__ float lerpf(float a, float b, float w) { return fmaf(w, b - a, a); }

// calc_sh (render_util.cuh:119-150) for basis_dim 9 at a unit world direction
__device__ __forceinline__ float sh_basis(const float d[3], int b) {
    const float x = d[0], y = d[1], z = d[2];
    switch (b) {
        case 0: return 0.28209479177387814f;
        case 1: return -0.4886025119029199f * y;
        case 2: return 0.4886025119029199f * z;
        case 3: return -0.4886025119029199f * x;
        case 4: return 1.0925484305920792f * (x * y);
        case 5: return -1.0925484305920792f * (y * z);
        case 6: return 0.31539156525252005f * (2.0f * (z * z) - (x * x) - (y * y));
        case 7: return -1.0925484305920792f * (x * z);
        default: return 0.5462742152960396f * ((x * x) - (y * y));
    }
}

// ray_find_bounds without the spheric clip and with near_clip 0 (render_util.cuh:253-311): moves the ray into grid coordinates with a
// unit direction; world_step is the world length of one step.  tmin > tmax: the ray misses the box.
__device__ __forceinline__ void find_bounds(Ray& r, const Grid& g, float step_size) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        r.o[j] = fmaf(r.o[j], g.scaling[j], g.offset[j]);
        r.d[j] *= g.scaling[j];
    }
    const float ds = rnorm3df(r.d[0], r.d[1], r.d[2]);
#pragma unroll
    for (int j = 0; j < 3; ++j) r.d[j] *= ds;
    r.world_step = ds * step_size;
    r.tmin = 0.f;
    r.tmax = 2e3f;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float inv = (float)(1.0 / r.d[j]);
        const float t1 = (-0.5f - r.o[j]) * inv, t2 = (g.size[j] - 0.5f - r.o[j]) * inv;
        if (r.d[j] != 0.f) {
            r.tmin = fmaxf(r.tmin, fminf(t1, t2));
            r.tmax = fminf(r.tmax, fmaxf(t1, t2));
        }
    }
}

// The cell of the sample at t: its lowest corner's linear index, and the fractional position p inside it.
__device__ __forceinline__ int locate(const int size[3], const float o[3], const float d[3], float t, float p[3]) {
    int l[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float x = fmaf(t, d[j], o[j]);
        x = fminf(fmaxf(x, 0.f), size[j] - 1.f);
        l[j] = min((int)x, size[j] - 2);
        p[j] = x - (float)l[j];
    }
    return (l[0] * size[1] + l[1]) * size[2] + l[2];
}

// corner k = (dx << 2) | (dy << 1) | dz of a cell: offset of its link from the cell's lowest corner
__device__ __forceinline__ int corner_offset(const int size[3], int k) {
    return ((k >> 2) & 1) * size[1] * size[2] + ((k >> 1) & 1) * size[2] + (k & 1);
}

// trilerp_cuvol_one's order of lerps over the 8 corner values
__device__ __forceinline__ float trilerp8(const float c[8], const float p[3]) {
    const float ix0 = lerpf(lerpf(c[0], c[1], p[2]), lerpf(c[2], c[3], p[2]), p[1]);
    const float ix1 = lerpf(lerpf(c[4], c[5], p[2]), lerpf(c[6], c[7], p[2]), p[1]);
    return lerpf(ix0, ix1, p[0]);
}

// trilerp_backward_cuvol_one's weight of corner k times g, in its order of products
__device__ __forceinline__ float corner_weight(const float p[3], int k, float g) {
    const float a = (k & 2) ? p[1] : 1.f - p[1];
    const float b = (k & 1) ? p[2] : 1.f - p[2];
    const float xo = (k & 4) ? p[0] * g : (1.f - p[0]) * g;
    return a * b * xo;
}

// Adds v to a fixed-point sum.  Integer addition is associative, so the sum does not depend on the order of the adds.  A term that is
// not finite or too large, or a sum that leaves the signed 64-bit range, sets *flag; the sum is then meaningless and the caller reports it.
__device__ __forceinline__ void fx_add(long long* addr, float v, unsigned* flag) {
    if (!(fabsf(v) < FX_MAX_TERM)) {
        atomicOr(flag, 1u);
        return;
    }
    const long long c = __float2ll_rn(v * FX_SCALE);
    if (c == 0) return;
    const unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)c);
    const long long o = (long long)old, n = (long long)(old + (unsigned long long)c);
    if (((o ^ n) & (c ^ n)) < 0) atomicOr(flag, 1u);
}
}  // namespace svox
