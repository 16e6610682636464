// Radial-tangential lens model of Instant-NGP / COLMAP captures (OpenCV's, with k3 = 0): the forward map from an undistorted normalised
// camera coordinate (x, y) -- camera frame x right, y down, z forward -- to the distorted one the pixel sees, and its inverse.
//   r2 = x^2 + y^2
//   x_d = x (1 + k1 r2 + k2 r2^2) + 2 p1 x y + p2 (r2 + 2 x^2)
//   y_d = y (1 + k1 r2 + k2 r2^2) + p1 (r2 + 2 y^2) + 2 p2 x y
// k = (k1, k2, p1, p2).  The reference reads these coefficients (dataset/dataset.py:123-126) and never applies them; the dataset's
// host-side check (plugin/dataset.py: check_lens) refuses lenses whose map folds over inside the image, so the solve below has a unique
// root to find.
#pragma once
#include <cuda_runtime.h>

__device__ __forceinline__ void lens_distort(float x, float y, float4 k, float& xd, float& yd) {
    const float r2 = x * x + y * y, rad = 1.f + r2 * (k.x + r2 * k.y);
    xd = x * rad + 2.f * k.z * x * y + k.w * (r2 + 2.f * x * x);
    yd = y * rad + k.z * (r2 + 2.f * y * y) + 2.f * k.w * x * y;
}

// In place: (x, y) distorted on entry, undistorted on exit.  Newton's method with the analytic 2x2 Jacobian, started at the distorted
// point, at most LENS_NEWTON_ITERS steps; it stops early once a step moves the point by less than LENS_NEWTON_TOL (a few fp32 ulps of a
// coordinate of order 1).
constexpr int LENS_NEWTON_ITERS = 10;
constexpr float LENS_NEWTON_TOL = 1e-7f;

__device__ __forceinline__ void lens_undistort(float& x, float& y, float4 k) {
    const float xt = x, yt = y;
#pragma unroll 1
    for (int it = 0; it < LENS_NEWTON_ITERS; ++it) {
        float fx, fy;
        lens_distort(x, y, k, fx, fy);
        fx -= xt;
        fy -= yt;
        const float r2 = x * x + y * y, rad = 1.f + r2 * (k.x + r2 * k.y), drad = 2.f * (k.x + 2.f * k.y * r2);   // d rad / d r2 times 2
        const float j11 = rad + x * x * drad + 2.f * k.z * y + 6.f * k.w * x;
        const float j22 = rad + y * y * drad + 6.f * k.z * y + 2.f * k.w * x;
        const float j12 = x * y * drad + 2.f * k.z * x + 2.f * k.w * y;                                               // = j21
        const float inv = 1.f / (j11 * j22 - j12 * j12);
        const float sx = (j22 * fx - j12 * fy) * inv, sy = (j11 * fy - j12 * fx) * inv;
        x -= sx;
        y -= sy;
        if (fabsf(sx) + fabsf(sy) < LENS_NEWTON_TOL) break;
    }
}
