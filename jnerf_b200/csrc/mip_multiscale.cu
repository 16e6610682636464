// The multiscale Mip-NeRF datasets of the reference's contrib/mipnerf (dataset/nerf.py: Blenders :207-314, Multicam :108-204) on the device:
// rays, targets and per-ray loss weights of global pixel ids over a ragged table of images of different sizes, and the fp32 encoder of the
// nn.Linear model at 8 or 16 IPE degrees (multicam.py: max_deg_point = 16).  Built with -fmad=false like mip_sampler.cu: the ray arithmetic
// is numpy's, and at degree 15 one contracted multiply-add in mip::gaussian moves an encoding column by ~1e-2.  DESIGN.md section 11.
#include "mip_common.cuh"
#include "ngp_b200.h"
#include "ngp_common.cuh"

namespace mip {
// A table row: pix2cam (3x3 row-major), cam2world (3x4 row-major), lossmult, near, far.
constexpr uint32_t CAM_FLOATS = 24;

__device__ __forceinline__ float texel(const uint8_t* p) { return (float)*p / 255.f; }
__device__ __forceinline__ float texel(const float* p) { return *p; }

// Multicam's direction: the pixel centre (x + .5, y + .5, 1) @ pix2cam^T @ cam2world[:3, :3]^T, each product term by term in index order.
__device__ __forceinline__ void pix_dir(const float* cam, float x, float y, float d[3]) {
    const float px = x + .5f, py = y + .5f;
    float c[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) c[j] = px * cam[3 * j] + py * cam[3 * j + 1] + 1.f * cam[3 * j + 2];
    const float* m = cam + 9;
#pragma unroll
    for (int j = 0; j < 3; ++j) d[j] = c[0] * m[4 * j] + c[1] * m[4 * j + 1] + c[2] * m[4 * j + 2];
}

// Global pixel p of image i = offsets[i] + y W_i + x, offsets (n_img + 1) ascending.  focal != 0 is Blenders (one focal length, the
// camera directions of cam_dir); focal = 0 is Multicam (the table's pix2cam).  Radius: |d(y) - d(y + 1)| * 2 / sqrt(12), the last row
// taking that of row H - 3 (dx[-2:-1]); target: rgb of the RGBA image, composited on white as rgb a + (1 - a) when `white`.
template <class Px>
__global__ void mip_rays_multi_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t n_img, const uint32_t* __restrict__ offsets,
                                      const uint32_t* __restrict__ wh, const float* __restrict__ cams, float focal, int white,
                                      const Px* __restrict__ images, float* __restrict__ rays, float* __restrict__ target,
                                      float* __restrict__ lossmult) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = pix[i];
    uint32_t lo = 0, hi = n_img;                                     // largest img with offsets[img] <= p
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (offsets[mid] <= p) lo = mid;
        else hi = mid;
    }
    const uint32_t img = lo, W = wh[2 * img], H = wh[2 * img + 1], q = p - offsets[img], y = q / W, x = q % W;
    const float* cam = cams + (size_t)img * CAM_FLOATS;
    const float* m = cam + 9;
    float d[3], a[3], b[3];
    const uint32_t y0 = y + 1 < H ? y : H - 3;
    if (focal != 0.f) {
        cam_dir(m, (float)x, (float)y, W, H, focal, d);
        cam_dir(m, (float)x, (float)y0, W, H, focal, a);
        cam_dir(m, (float)x, (float)(y0 + 1), W, H, focal, b);
    } else {
        pix_dir(cam, (float)x, (float)y, d);
        pix_dir(cam, (float)x, (float)y0, a);
        pix_dir(cam, (float)x, (float)(y0 + 1), b);
    }
    const float e0 = a[0] - b[0], e1 = a[1] - b[1], e2 = a[2] - b[2];
    const float dx = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
    const float norm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    float* r = rays + (size_t)i * RAY_FLOATS;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        r[j] = m[4 * j + 3];
        r[3 + j] = d[j];
        r[6 + j] = d[j] / norm;
    }
    r[9] = (float)((double)(dx * 2.f) / 3.4641016151377544);
    r[10] = cam[22];
    r[11] = cam[23];
    const Px* px = images + (size_t)p * 4;
    const float alpha = texel(px + 3);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float c = texel(px + j);
        target[(size_t)i * 3 + j] = white ? c * alpha + (1.f - alpha) : c;
    }
    lossmult[i] = cam[21];
}

// fp32 encoder of the nn.Linear model: IPE (N, 6 DEGS) and pos_enc(viewdir, 0, 4) (N, 27), both in the reference's column orders
template <uint32_t DEGS>
__global__ void mip_encode_deg_kernel(uint32_t N, uint32_t S, const float* __restrict__ rays, const float* __restrict__ t, int cylinder,
                                      int integrate, int min_deg, float* __restrict__ enc, float* __restrict__ view) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= N * 3) return;
    const uint32_t row = k / 3, dim = k % 3, ray = row / S, i = row % S;
    const float* ry = rays + (size_t)ray * RAY_FLOATS;
    const float* tt = t + (size_t)ray * (S + 1) + i;
    float mean, var;
    gaussian(ry, tt[0], tt[1], dim, cylinder, integrate, mean, var);
    float* e = enc + (size_t)row * 6 * DEGS;
    ipe<DEGS>(mean, var, dim, min_deg, [&](uint32_t f, float v) { e[f] = v; });
    float* o = view + (size_t)row * (3 + 6 * VIEW_DEGS);
    const float x = ry[6 + dim];
    o[dim] = x;
#pragma unroll
    for (uint32_t q = 0; q < VIEW_DEGS; ++q) {
        float sn, cs;
        sincosf(x * (float)(1u << q), &sn, &cs);
        o[3 + 3 * q + dim] = sn;
        o[3 + 3 * VIEW_DEGS + 3 * q + dim] = cs;
    }
}
}  // namespace mip

using namespace mip;

extern "C" {

int ngp_mip_rays_multi(void* stream, uint32_t n, const uint32_t* pix, uint32_t n_images, const uint32_t* offsets, const uint32_t* wh,
                       const float* cams, float focal, int white_bkgd, const void* images_rgba, int float_images, float* rays_out, float* target_out,
                       float* lossmult_out) {
    if (n == 0) return 0;
    NGP_REQUIRE(n_images >= 1, "ngp_mip_rays_multi: no images");
    NGP_REQUIRE(pix && offsets && wh && cams && images_rgba && rays_out && target_out && lossmult_out, "ngp_mip_rays_multi: NULL input");
    const uint32_t b = (n + 255) / 256;
    cudaStream_t s = (cudaStream_t)stream;
    if (!float_images)
        mip_rays_multi_kernel<uint8_t><<<b, 256, 0, s>>>(n, pix, n_images, offsets, wh, cams, focal, white_bkgd, (const uint8_t*)images_rgba, rays_out,
                                                         target_out, lossmult_out);
    else
        mip_rays_multi_kernel<float><<<b, 256, 0, s>>>(n, pix, n_images, offsets, wh, cams, focal, white_bkgd, (const float*)images_rgba, rays_out,
                                                       target_out, lossmult_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_encode_deg(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate,
                       int min_deg, int degs, float* enc_out, float* view_out) {
    NGP_REQUIRE(degs == 8 || degs == 16, "ngp_mip_encode_deg: degs must be 8 or 16");
    NGP_REQUIRE(n_samples >= 1 && (uint64_t)n_rays * n_samples * 3 < (1ull << 32),
                "ngp_mip_encode_deg: n_samples must be >= 1, n_rays * n_samples < 2^32 / 3");
    NGP_REQUIRE(ray_shape == 0 || ray_shape == 1, "ngp_mip_encode_deg: ray_shape must be 0 (cone) or 1 (cylinder)");
    const uint32_t N = n_rays * n_samples;
    if (N == 0) return 0;
    NGP_REQUIRE(rays && t && enc_out && view_out, "ngp_mip_encode_deg: NULL input");
    const uint32_t b = (uint32_t)(((uint64_t)N * 3 + 255) / 256);
    cudaStream_t s = (cudaStream_t)stream;
    if (degs == 16)
        mip_encode_deg_kernel<16><<<b, 256, 0, s>>>(N, n_samples, rays, t, ray_shape, integrate != 0, min_deg, enc_out, view_out);
    else
        mip_encode_deg_kernel<8><<<b, 256, 0, s>>>(N, n_samples, rays, t, ray_shape, integrate != 0, min_deg, enc_out, view_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
