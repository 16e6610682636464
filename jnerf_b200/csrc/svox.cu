// Plenoxels (the svox2 port under the reference's contrib/plenoxel): training step, whole-frame rendering, sparse total variation,
// RMSprop and the kernels of the prune-and-upsample pass.  All fp32.  Gradients are sums of signed 64-bit fixed-point terms added with
// integer atomics, so a training step gives the same bits whatever the order the warps run in; the one float atomic-free max
// (weight_render) is order-independent too.  DESIGN.md section 12.
#include "mesh_scan.cuh"
#include "ngp_b200.h"
#include "ngp_common.cuh"
#include "svox_common.cuh"

namespace svox {
namespace {
constexpr uint32_t WARPS = 8;              // rays per 256-thread block of the warp-per-ray kernels

__host__ __device__ inline uint32_t blocks(uint64_t n, uint32_t per) { return (uint32_t)((n + per - 1) / per); }

// Pixel (img * H + y) * W + x of a camera with intrinsics (fx, fy, cx, cy) and OpenCV camera-to-world c2w (3x4 row-major) -> world ray
// through the pixel centre with a unit direction (svox_dataset.py gen_rays, svox2_utils.py Camera.gen_rays).
__device__ __forceinline__ void pixel_ray(const float* c2w, float fx, float fy, float cx, float cy, uint32_t x, uint32_t y, Ray& r) {
    const float u = ((float)x + 0.5f - cx) / fx, v = ((float)y + 0.5f - cy) / fy;
    const float inv = 1.f / sqrtf(u * u + v * v + 1.f);
    const float a = u * inv, b = v * inv, c = inv;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        r.o[j] = c2w[4 * j + 3];
        r.d[j] = c2w[4 * j] * a + c2w[4 * j + 1] * b + c2w[4 * j + 2] * c;
    }
}

// One sample's corner links and densities, loaded by lanes 0-7 (one corner each) and broadcast; returns sigma.
__device__ __forceinline__ float sample_sigma(const Grid& g, int base, int coff, const float p[3], int L[8]) {
    const int lk = g.links[base + coff];
    const float dv = lk >= 0 ? g.density[lk] : 0.f;
    float c[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        c[k] = __shfl_sync(FULL, dv, k);
        L[k] = __shfl_sync(FULL, lk, k);
    }
    return trilerp8(c, p);
}

// The lane's SH coefficient (lane < 27: channel lane / 9, basis lane % 9) trilerped at the sample.
__device__ __forceinline__ float sample_coeff(const Grid& g, const int L[8], const float p[3], uint32_t lane) {
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = (L[k] >= 0 && lane < DATA_DIM) ? g.sh[(size_t)L[k] * DATA_DIM + lane] : 0.f;
    return trilerp8(s, p);
}

// Sum of v over the 9 lanes of this lane's channel group (lanes 27-31 get garbage).
__device__ __forceinline__ float group_sum(float v, uint32_t lane) {
    const uint32_t g0 = lane / BASIS * BASIS;
    float s = 0.f;
#pragma unroll
    for (int b = 0; b < BASIS; ++b) s += __shfl_sync(FULL, v, (g0 + b) & 31);
    return s;
}

// trace_ray_cuvol (volume_render_cuvol_fused.h:41-149) by one warp: every lane of channel group c returns channel c of the colour,
// background included.  r has been through find_bounds.
__device__ float march_forward(const Grid& g, const Opt& opt, const Ray& r, float sph, uint32_t lane) {
    if (r.tmin > r.tmax) return opt.background;
    const int coff = corner_offset(g.size, lane & 7);
    float outv = 0.f, log_t = 0.f;
    for (float t = r.tmin; t <= r.tmax; t += opt.step_size) {
        float p[3];
        int L[8];
        const int base = locate(g.size, r.o, r.d, t, p);
        const float sigma = sample_sigma(g, base, coff, p, L);
        if (sigma > opt.sigma_thresh) {
            const float tot = group_sum(sample_coeff(g, L, p, lane) * sph, lane);
            const float pcnt = r.world_step * sigma;
            const float weight = __expf(log_t) * (1.f - __expf(-pcnt));
            log_t -= pcnt;
            outv += weight * fmaxf(tot + 0.5f, 0.f);
            if (__expf(log_t) < opt.stop_thresh) {
                log_t = -1e3f;
                break;
            }
        }
    }
    return outv + __expf(log_t) * opt.background;
}

__device__ __forceinline__ void pixel_of(uint32_t pix, uint32_t W, uint32_t H, uint32_t& img, uint32_t& x, uint32_t& y) {
    img = pix / (W * H);
    y = (pix / W) % H;
    x = pix % W;
}

// ---- training step: forward, MSE gradient, re-marched backward (render_ray_backward_kernel, :207-460), one warp a ray -------------
__global__ void __launch_bounds__(32 * WARPS) train_step_kernel(uint32_t R, const int32_t* __restrict__ pix, uint32_t W, uint32_t H,
                                                                const float* __restrict__ c2w, float fx, float fy, float cx, float cy,
                                                                const uint8_t* __restrict__ images, Grid g, Opt opt, long long* __restrict__ gd,
                                                                long long* __restrict__ gs, float* __restrict__ sqerr, unsigned* __restrict__ flag) {
    const uint32_t ray = blockIdx.x * WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (ray >= R) return;
    uint32_t img, x, y;
    pixel_of((uint32_t)pix[ray], W, H, img, x, y);
    Ray r;
    pixel_ray(c2w + (size_t)img * 12, fx, fy, cx, cy, x, y, r);
    const float sph = sh_basis(r.d, lane % BASIS);
    find_bounds(r, g, opt.step_size);
    const float col = march_forward(g, opt, r, sph, lane);
    float rgb[3], gout[3];
    const uint8_t* px = images + ((size_t)img * H * W + (size_t)y * W + x) * 4;
    const float alpha = (float)px[3] / 255.f;
    const float norm = 2.f / (3.f * (float)R);
    float se = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        rgb[c] = __shfl_sync(FULL, col, BASIS * c);
        const float gt = (float)px[c] / 255.f * alpha + (1.f - alpha);
        const float d = rgb[c] - gt;
        se += d * d;
        gout[c] = d * norm;
    }
    if (lane == 0) sqerr[ray] = se;
    if (r.tmin > r.tmax) return;
    const uint32_t ch = min(lane / BASIS, 2u);
    const float my_gout = ch == 0 ? gout[0] : ch == 1 ? gout[1] : gout[2];
    float accum = fmaf(rgb[0], gout[0], fmaf(rgb[1], gout[1], rgb[2] * gout[2]));
    const int coff = corner_offset(g.size, lane & 7);
    float log_t = 0.f;
    for (float t = r.tmin; t <= r.tmax; t += opt.step_size) {
        float p[3];
        int L[8];
        const int base = locate(g.size, r.o, r.d, t, p);
        const float sigma = sample_sigma(g, base, coff, p, L);
        if (sigma > opt.sigma_thresh) {
            const float tot = group_sum(sample_coeff(g, L, p, lane) * sph, lane) + 0.5f;
            const float pcnt = r.world_step * sigma;
            const float weight = __expf(log_t) * (1.f - __expf(-pcnt));
            log_t -= pcnt;
            float total_color = fmaxf(tot, 0.f);
            const float in01 = total_color == tot ? 1.f : 0.f;
            total_color *= my_gout;
            const float c1 = __shfl_sync(FULL, total_color, BASIS);
            const float tc = (__shfl_sync(FULL, total_color, 0) + __shfl_sync(FULL, total_color, 2 * BASIS)) + c1;
            const float grad_color = sph * (weight * in01 * my_gout);
            accum -= weight * tc;
            const float grad_sigma = r.world_step * (tc * __expf(log_t) - accum);
            if (lane < DATA_DIM) {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (L[k] >= 0) fx_add(gs + (size_t)L[k] * DATA_DIM + lane, corner_weight(p, k, grad_color), flag);
            }
            if (lane >= 24) {
                const int k = lane - 24;                                  // lanes 24-31 add the density term of corner lane - 24
                int lk = L[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) lk = j == k ? L[j] : lk;
                if (lk >= 0) fx_add(gd + lk, corner_weight(p, k, grad_sigma), flag);
            }
            if (__expf(log_t) < opt.stop_thresh) break;
        }
    }
}

// ---- whole-frame rendering: pixels [first, first + n) of one camera --------------------------------------------------------------
__global__ void __launch_bounds__(32 * WARPS) render_kernel(uint32_t n, uint32_t first, uint32_t W, const float* __restrict__ c2w, float fx, float fy,
                                                            float cx, float cy, Grid g, Opt opt, float* __restrict__ rgb_out) {
    const uint32_t i = blockIdx.x * WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint32_t pix = first + i;
    Ray r;
    pixel_ray(c2w, fx, fy, cx, cy, pix % W, pix / W, r);
    const float sph = sh_basis(r.d, lane % BASIS);
    find_bounds(r, g, opt.step_size);
    const float col = march_forward(g, opt, r, sph, lane);
    if (lane % BASIS == 0 && lane < DATA_DIM) rgb_out[(size_t)i * 3 + lane / BASIS] = col;
}

// ---- sparse TV (tv_grad_sparse_kernel, loss_kernel.h:51-118): cells (start + i) mod (X Y Z), i < n_cells, columns [0, dim) ----------
__global__ void tv_kernel(uint64_t Q, uint32_t dim, uint32_t start, uint32_t n_cells, const int32_t* __restrict__ links, int X, int Y, int Z,
                          const float* __restrict__ data, float scale, int ignore_edge, long long* __restrict__ grad, unsigned* __restrict__ flag) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= Q) return;
    const uint32_t idx = (uint32_t)(tid % dim);
    const uint64_t G = (uint64_t)X * Y * Z;
    const int xyz = (int)(((uint64_t)start + tid / dim) % G);
    const int z = xyz % Z, xy = xyz / Z, y = xy % Y, x = xy / Y;
    const int32_t* lp = links + xyz;
    if (ignore_edge && *lp == 0) return;
    const float s0 = X * (1.f / 256.f), s1 = Y * (1.f / 256.f), s2 = Z * (1.f / 256.f);
    const int32_t l000 = lp[0];
    const int32_t l001 = z + 1 < Z ? lp[1] : 0;
    const int32_t l010 = y + 1 < Y ? lp[Z] : 0;
    const int32_t l100 = x + 1 < X ? lp[Y * Z] : 0;
    const float v000 = l000 >= 0 ? data[(size_t)l000 * dim + idx] : 0.f;
    const float nul = ignore_edge ? v000 : 0.f;
    const float v001 = l001 >= 0 ? data[(size_t)l001 * dim + idx] : nul;
    const float v010 = l010 >= 0 ? data[(size_t)l010 * dim + idx] : nul;
    const float v100 = l100 >= 0 ? data[(size_t)l100 * dim + idx] : nul;
    float dx = v100 - v000, dy = v010 - v000, dz = v001 - v000;
    const float idelta = scale * rsqrtf(1e-9f + dx * dx + dy * dy + dz * dz);
    dx *= s0;
    dy *= s1;
    dz *= s2;
    const float sm = -(dx + dy + dz);
    if (l000 >= 0 && sm != 0.f) fx_add(grad + (size_t)l000 * dim + idx, sm * idelta, flag);
    if (l001 >= 0 && dz != 0.f) fx_add(grad + (size_t)l001 * dim + idx, dz * idelta, flag);
    if (l010 >= 0 && dy != 0.f) fx_add(grad + (size_t)l010 * dim + idx, dy * idelta, flag);
    if (l100 >= 0 && dx != 0.f) fx_add(grad + (size_t)l100 * dim + idx, dx * idelta, flag);
}

// ---- RMSprop over density (n_d entries) then SH (n_s entries); the fixed-point gradient read is cleared -----------------------------
// One thread a chunk of 4 consecutive entries of one tensor (16-byte parameter / state loads, two 16-byte gradient loads); a tensor's
// last chunk may be partial.
__device__ __forceinline__ float rms_one(float& p, float& v, long long& g, float lr, float a, float eps) {
    const float gr = __ll2float_rn(g) * FX_UNIT;
    g = 0;
    v = a * v + (1.f - a) * gr * gr;
    p = p - lr * gr / (sqrtf(v) + eps);
    return p;
}

__global__ void __launch_bounds__(256) rmsprop_kernel(uint64_t n_d, uint64_t n_s, float* __restrict__ pd, float* __restrict__ ps,
                                                      long long* __restrict__ gd, long long* __restrict__ gs, float* __restrict__ vd,
                                                      float* __restrict__ vs, float lr_d, float lr_s, float alpha_d, float alpha_s, float eps) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, cd = (n_d + 3) / 4;
    const bool den = c < cd;
    const uint64_t n = den ? n_d : n_s, j = 4 * (den ? c : c - cd);
    if (j >= n) return;
    float* p = (den ? pd : ps) + j;
    float* v = (den ? vd : vs) + j;
    long long* g = (den ? gd : gs) + j;
    const float lr = den ? lr_d : lr_s, a = den ? alpha_d : alpha_s;
    if (j + 4 <= n && ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(g)) & 15) == 0) {
        float4 P = *reinterpret_cast<float4*>(p), V = *reinterpret_cast<float4*>(v);
        longlong2 G0 = reinterpret_cast<longlong2*>(g)[0], G1 = reinterpret_cast<longlong2*>(g)[1];
        rms_one(P.x, V.x, G0.x, lr, a, eps);
        rms_one(P.y, V.y, G0.y, lr, a, eps);
        rms_one(P.z, V.z, G1.x, lr, a, eps);
        rms_one(P.w, V.w, G1.y, lr, a, eps);
        *reinterpret_cast<float4*>(p) = P;
        *reinterpret_cast<float4*>(v) = V;
        reinterpret_cast<longlong2*>(g)[0] = G0;
        reinterpret_cast<longlong2*>(g)[1] = G1;
    } else {
        for (uint64_t k = 0; k < 4 && j + k < n; ++k) rms_one(p[k], v[k], g[k], lr, a, eps);
    }
}

// ---- resample: trilerp at points in grid coordinates (sample_kernel.h); column 0 density, 1-27 SH --------------------------------
__global__ void sample_kernel(uint64_t Q, uint32_t cols, const float* __restrict__ pts, Grid g, float* __restrict__ dens_out,
                              float* __restrict__ sh_out) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= Q) return;
    const uint32_t col = (uint32_t)(tid % cols);
    const uint64_t i = tid / cols;
    float p[3];
    const float o[3] = {pts[i * 3], pts[i * 3 + 1], pts[i * 3 + 2]}, d[3] = {0.f, 0.f, 0.f};
    const int base = locate(g.size, o, d, 0.f, p);
    float c[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int lk = g.links[base + corner_offset(g.size, k)];
        c[k] = lk < 0 ? 0.f : col == 0 ? g.density[lk] : g.sh[(size_t)lk * DATA_DIM + col - 1];
    }
    const float v = trilerp8(c, p);
    if (col == 0)
        dens_out[i] = v;
    else
        sh_out[i * DATA_DIM + col - 1] = v;
}

// ---- resample: max weight of each cell of a dense density grid over one camera's rays (grid_weight_render_kernel, misc_kernel.h) ---
__global__ void weight_render_kernel(uint32_t W, uint32_t H, const float* __restrict__ c2w, float fx, float fy, float cx, float cy,
                                     const float* __restrict__ data, Grid g, float step_size, float stop_thresh, float* __restrict__ out) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= W * H) return;
    const uint32_t ix = tid % W, iy = tid / W;
    float x = ((float)ix + 0.5f - cx) / fx, y = ((float)iy + 0.5f - cy) / fy;
    float z = sqrtf((float)((double)(x * x + y * y) + 1.0));
    x /= z;
    y /= z;
    z = 1.0f / z;
    Ray r;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        r.d[j] = c2w[4 * j] * x + c2w[4 * j + 1] * y + c2w[4 * j + 2] * z;
        r.o[j] = c2w[4 * j + 3];
    }
    find_bounds(r, g, step_size);
    if (r.tmin > r.tmax) return;
    const int s1 = g.size[2], s0 = g.size[1] * g.size[2];
    float log_t = 0.f;
    for (float t = r.tmin; t <= r.tmax; t += step_size) {
        float p[3];
        const int idx = locate(g.size, r.o, r.d, t, p);
        const float* a = data + idx;
        const float* b = a + s0;
        const float sigma = lerpf(lerpf(lerpf(a[0], a[1], p[2]), lerpf(a[s1], a[s1 + 1], p[2]), p[1]),
                                  lerpf(lerpf(b[0], b[1], p[2]), lerpf(b[s1], b[s1 + 1], p[2]), p[1]), p[0]);
        if (sigma > 1e-8f) {
            const float att = -r.world_step * sigma;
            // clamped to >= 0 (__expf may round a factor to one ulp past 1): the order of non-negative floats is the order of their bits
            // as unsigned integers, and a max does not depend on the order of the updates
            const float w = fmaxf(__expf(log_t) * (1.f - __expf(att)), 0.f);
            log_t += att;
            const unsigned wu = __float_as_uint(w);
            unsigned* m = reinterpret_cast<unsigned*>(out + idx);
            atomicMax(m, wu);
            atomicMax(m + 1, wu);
            atomicMax(m + s1, wu);
            atomicMax(m + s1 + 1, wu);
            atomicMax(m + s0, wu);
            atomicMax(m + s0 + 1, wu);
            atomicMax(m + s0 + s1, wu);
            atomicMax(m + s0 + s1 + 1, wu);
            if (__expf(log_t) < stop_thresh) break;
        }
    }
}

// ---- resample: 26-neighbourhood dilation of a uint8 mask (dilate_kernel, misc_kernel.h:11-39) -------------------------------------
__global__ void dilate_kernel(int X, int Y, int Z, const uint8_t* __restrict__ in, uint8_t* __restrict__ out) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (uint64_t)X * Y * Z) return;
    const int z = (int)(tid % Z), y = (int)(tid / Z % Y), x = (int)(tid / ((uint64_t)Y * Z));
    uint8_t v = 0;
    for (int i = max(x - 1, 0); i <= min(x + 1, X - 1); ++i)
        for (int j = max(y - 1, 0); j <= min(y + 1, Y - 1); ++j)
            for (int k = max(z - 1, 0); k <= min(z + 1, Z - 1); ++k) v |= in[((size_t)i * Y + j) * Z + k] != 0;
    out[tid] = v;
}

__global__ void mask_to_u32_kernel(uint64_t n, const uint8_t* __restrict__ mask, uint32_t* __restrict__ a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = mask[i] != 0;
}

// kept cell i (its exclusive count c = a[i]) -> link c, density c = dense[i], point c = the cell's centre in the old grid's coordinates
__global__ void compact_kernel(int X, int Y, int Z, const uint8_t* __restrict__ mask, const uint32_t* __restrict__ a, const float* __restrict__ dense,
                               float s0, float s1, float s2, float d0, float d1, float d2, uint32_t capacity, int32_t* __restrict__ links,
                               float* __restrict__ dens_out, float* __restrict__ pts_out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)X * Y * Z) return;
    if (!mask[i]) {
        links[i] = -1;
        return;
    }
    const uint32_t c = a[i];
    links[i] = (int32_t)c;
    if (c >= capacity) return;
    const int z = (int)(i % Z), y = (int)(i / Z % Y), x = (int)(i / ((uint64_t)Y * Z));
    dens_out[c] = dense[i];
    pts_out[(size_t)c * 3] = s0 + (float)x * d0;
    pts_out[(size_t)c * 3 + 1] = s1 + (float)y * d1;
    pts_out[(size_t)c * 3 + 2] = s2 + (float)z * d2;
}

Grid make_grid(const int32_t* links, int X, int Y, int Z, const float* density, const float* sh, const float* xform) {
    Grid g{links, density, sh, {X, Y, Z}, {0.f, 0.f, 0.f}, {1.f, 1.f, 1.f}};
    if (xform)
        for (int j = 0; j < 3; ++j) {
            g.offset[j] = xform[j];
            g.scaling[j] = xform[3 + j];
        }
    return g;
}
}  // namespace
}  // namespace svox

using namespace svox;

extern "C" {

int ngp_svox_train_step(void* stream, uint32_t n_rays, const int32_t* pix, uint32_t W, uint32_t H, const float* c2w, float fx, float fy, float cx,
                        float cy, const uint8_t* images_rgba, const int32_t* links, int X, int Y, int Z, const float* density, const float* sh,
                        const float* xform, const float* opts, long long* grad_density, long long* grad_sh, float* sqerr_out, unsigned* flag) {
    NGP_REQUIRE(X >= 2 && Y >= 2 && Z >= 2 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_train_step: grid sides must be >= 2, X Y Z < 2^31");
    NGP_REQUIRE(xform && opts, "ngp_svox_train_step: xform / opts (host arrays) must be given");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(pix && c2w && images_rgba && links && density && sh && grad_density && grad_sh && sqerr_out && flag, "ngp_svox_train_step: NULL input");
    const Grid g = make_grid(links, X, Y, Z, density, sh, xform);
    const Opt opt{opts[0], opts[1], opts[2], opts[3]};
    train_step_kernel<<<blocks(n_rays, WARPS), 32 * WARPS, 0, (cudaStream_t)stream>>>(n_rays, pix, W, H, c2w, fx, fy, cx, cy, images_rgba, g, opt,
                                                                                        grad_density, grad_sh, sqerr_out, flag);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_render(void* stream, uint32_t n, uint32_t first, uint32_t W, const float* c2w, float fx, float fy, float cx, float cy, const int32_t* links,
                    int X, int Y, int Z, const float* density, const float* sh, const float* xform, const float* opts, float* rgb_out) {
    NGP_REQUIRE(X >= 2 && Y >= 2 && Z >= 2 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_render: grid sides must be >= 2, X Y Z < 2^31");
    NGP_REQUIRE(xform && opts && W > 0, "ngp_svox_render: xform / opts (host arrays) and W > 0 must be given");
    if (n == 0) return 0;
    NGP_REQUIRE(c2w && links && density && sh && rgb_out, "ngp_svox_render: NULL input");
    const Grid g = make_grid(links, X, Y, Z, density, sh, xform);
    const Opt opt{opts[0], opts[1], opts[2], opts[3]};
    render_kernel<<<blocks(n, WARPS), 32 * WARPS, 0, (cudaStream_t)stream>>>(n, first, W, c2w, fx, fy, cx, cy, g, opt, rgb_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_tv_grad(void* stream, const int32_t* links, int X, int Y, int Z, const float* data, uint32_t dim, uint32_t start, uint32_t n_cells,
                     float scale, int ignore_edge, long long* grad, unsigned* flag) {
    NGP_REQUIRE(X >= 1 && Y >= 1 && Z >= 1 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_tv_grad: X Y Z must be in [1, 2^31)");
    NGP_REQUIRE(dim >= 1 && start < (uint64_t)X * Y * Z && n_cells <= (uint64_t)X * Y * Z, "ngp_svox_tv_grad: dim >= 1, start and n_cells within the grid");
    if (n_cells == 0) return 0;
    NGP_REQUIRE(links && data && grad && flag, "ngp_svox_tv_grad: NULL input");
    const uint64_t Q = (uint64_t)n_cells * dim;
    tv_kernel<<<blocks(Q, 256), 256, 0, (cudaStream_t)stream>>>(Q, dim, start, n_cells, links, X, Y, Z, data, scale, ignore_edge, grad, flag);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_rmsprop(void* stream, uint64_t n_density, uint64_t n_sh, float* density, float* sh, long long* grad_density, long long* grad_sh,
                     float* rms_density, float* rms_sh, float lr_density, float lr_sh, float alpha_density, float alpha_sh, float eps) {
    if (n_density + n_sh == 0) return 0;
    NGP_REQUIRE(density && grad_density && rms_density && (n_sh == 0 || (sh && grad_sh && rms_sh)), "ngp_svox_rmsprop: NULL input");
    const uint64_t chunks = (n_density + 3) / 4 + (n_sh + 3) / 4;
    NGP_REQUIRE(chunks < (1ull << 31) * 256, "ngp_svox_rmsprop: too many entries");
    rmsprop_kernel<<<blocks(chunks, 256), 256, 0, (cudaStream_t)stream>>>(n_density, n_sh, density, sh, grad_density, grad_sh, rms_density, rms_sh, lr_density, lr_sh,
                                                        alpha_density, alpha_sh, eps);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_sample(void* stream, uint32_t n, const float* points, const int32_t* links, int X, int Y, int Z, const float* density, const float* sh,
                    int want_sh, float* density_out, float* sh_out) {
    NGP_REQUIRE(X >= 2 && Y >= 2 && Z >= 2 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_sample: grid sides must be >= 2, X Y Z < 2^31");
    if (n == 0) return 0;
    NGP_REQUIRE(points && links && density && density_out && (!want_sh || (sh && sh_out)), "ngp_svox_sample: NULL input");
    const uint32_t cols = want_sh ? 1 + DATA_DIM : 1;
    const Grid g = make_grid(links, X, Y, Z, density, sh, nullptr);
    const uint64_t Q = (uint64_t)n * cols;
    sample_kernel<<<blocks(Q, 256), 256, 0, (cudaStream_t)stream>>>(Q, cols, points, g, density_out, sh_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_weight_render(void* stream, uint32_t W, uint32_t H, const float* c2w, float fx, float fy, float cx, float cy, const float* data, int X, int Y,
                           int Z, const float* xform, float step_size, float stop_thresh, float* weight_out) {
    NGP_REQUIRE(X >= 2 && Y >= 2 && Z >= 2 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_weight_render: grid sides must be >= 2, X Y Z < 2^31");
    NGP_REQUIRE(xform && step_size > 0.f, "ngp_svox_weight_render: xform (host array) and step_size > 0 must be given");
    if ((uint64_t)W * H == 0) return 0;
    NGP_REQUIRE(c2w && data && weight_out, "ngp_svox_weight_render: NULL input");
    const Grid g = make_grid(nullptr, X, Y, Z, nullptr, nullptr, xform);
    weight_render_kernel<<<blocks((uint64_t)W * H, 256), 256, 0, (cudaStream_t)stream>>>(W, H, c2w, fx, fy, cx, cy, data, g, step_size, stop_thresh,
                                                                                         weight_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_dilate(void* stream, int X, int Y, int Z, const uint8_t* mask, uint8_t* out) {
    NGP_REQUIRE(X >= 1 && Y >= 1 && Z >= 1 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_dilate: X Y Z must be in [1, 2^31)");
    NGP_REQUIRE(mask && out && mask != out, "ngp_svox_dilate: NULL or aliased input");
    const uint64_t n = (uint64_t)X * Y * Z;
    dilate_kernel<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(X, Y, Z, mask, out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_svox_compact_workspace_bytes(int X, int Y, int Z, uint64_t* bytes_out) {
    NGP_REQUIRE(X >= 1 && Y >= 1 && Z >= 1 && (uint64_t)X * Y * Z < (1ull << 31) && bytes_out, "ngp_svox_compact_workspace_bytes: bad size");
    const uint64_t n = (uint64_t)X * Y * Z;
    *bytes_out = 4 * (n + blocks(n, ngp_mesh::SCAN_BLOCK) + 1);
    return 0;
}

int ngp_svox_compact(void* stream, int X, int Y, int Z, const uint8_t* mask, const float* dense_density, const float* lattice, uint32_t capacity,
                     void* workspace, int32_t* links_out, float* density_out, float* points_out) {
    NGP_REQUIRE(X >= 1 && Y >= 1 && Z >= 1 && (uint64_t)X * Y * Z < (1ull << 31), "ngp_svox_compact: X Y Z must be in [1, 2^31)");
    NGP_REQUIRE(lattice, "ngp_svox_compact: lattice (host array) must be given");
    NGP_REQUIRE(mask && dense_density && workspace && links_out && (capacity == 0 || (density_out && points_out)), "ngp_svox_compact: NULL input");
    cudaStream_t s = (cudaStream_t)stream;
    const uint64_t n = (uint64_t)X * Y * Z;
    uint32_t* a = (uint32_t*)workspace;
    uint32_t* bsum = a + n;
    uint32_t* total = bsum + blocks(n, ngp_mesh::SCAN_BLOCK);
    mask_to_u32_kernel<<<blocks(n, 256), 256, 0, s>>>(n, mask, a);
    NGP_LAUNCH_CHECK();
    if (ngp_mesh::scan_u32(s, a, (uint32_t)n, bsum, total)) return 1;
    compact_kernel<<<blocks(n, 256), 256, 0, s>>>(X, Y, Z, mask, a, dense_density, lattice[0], lattice[1], lattice[2], lattice[3], lattice[4],
                                                  lattice[5], capacity, links_out, density_out, points_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
