// Mip-NeRF's sampler around the network (MipSampler, models/samplers/mip_sampler/mip_sampler.py, and utils/miputils.py of the reference's
// contrib/mipnerf): per-batch ray generation of the Blender dataset, stratified fenceposts, hierarchical resampling from the blurred coarse
// weights, the fp32 encoder of the nn.Linear model, and the composite forward / loss backward.  Every kernel is fp32 and per ray, with no
// float atomics: the results do not depend on scheduling.  Uniforms come from pcg32: the kernel drawing n_per_ray of them a ray gives ray g
// the draws [g * n_per_ray, (g + 1) * n_per_ray) of the stream at (rng_state, rng_inc), in index order.  DESIGN.md section 11.
#include "mip_common.cuh"
#include "ngp_b200.h"
#include "ngp_common.cuh"

namespace mip {
constexpr uint32_t WARPS = 8;              // rays per 256-thread block of the warp-per-ray kernels
constexpr float EPS32 = 1.1920928955078125e-07f;   // np.finfo(float32).eps

__device__ __forceinline__ float ld(const float* p) { return *p; }
__device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ void st(float* p, float v) { *p = v; }
__device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// inclusive prefix sum over the lanes
__device__ __forceinline__ float warp_scan(float v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= (uint32_t)o) v += u;
    }
    return v;
}

// ---- Blender rays (dataset/nerf_datasets.py:193-235) ---------------------------------------------------------------------------------
// Pixel p = (img * H + y) * W + x.  camera_dirs = [(x - W/2 + 0.5) / f, -(y - H/2 + 0.5) / f, -1], direction = camera_dirs @ R^T, radius
// = |direction(y) - direction(y + 1)| * 2 / sqrt(12) (the last row takes that of row H - 3, as dx[-2:-1] does), all in fp32 in the order
// numpy evaluates them (this file is built with -fmad=false); the division by sqrt(12) in fp64, as numpy promotes it.  cam_dir is in
// mip_common.cuh.
__global__ void mip_rays_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t W, uint32_t H, const float* __restrict__ c2w, float focal,
                                float near, float far, const uint8_t* __restrict__ images, float* __restrict__ rays, float* __restrict__ target) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = pix[i], img = p / (W * H), y = (p / W) % H, x = p % W;
    const float* m = c2w + (size_t)img * 12;
    float d[3], a[3], b[3];
    cam_dir(m, (float)x, (float)y, W, H, focal, d);
    const uint32_t y0 = y + 1 < H ? y : H - 3;                       // dx[-2:-1] of :231 for the last row; H >= 3
    cam_dir(m, (float)x, (float)y0, W, H, focal, a);
    cam_dir(m, (float)x, (float)(y0 + 1), W, H, focal, b);
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
    r[10] = near;
    r[11] = far;
    const uint8_t* px = images + (size_t)p * 4;
#pragma unroll
    for (int j = 0; j < 3; ++j) target[(size_t)i * 3 + j] = (float)px[j] / 255.f;
}

// ---- stratified fenceposts (sample_along_rays, miputils.py:324-362) --------------------------------------------------------------------
__global__ void mip_sample_kernel(uint32_t R, uint32_t S, const float* __restrict__ rays, int lindisp, int randomized, Pcg32 rng,
                                  float* __restrict__ t_out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= R) return;
    const float near = rays[(size_t)g * RAY_FLOATS + 10], far = rays[(size_t)g * RAY_FLOATS + 11];
    auto fence = [&](uint32_t j) {
        const float v = (float)j / (float)S;
        return lindisp ? 1.f / (1.f / near * (1.f - v) + 1.f / far * v) : near + (far - near) * v;
    };
    float* out = t_out + (size_t)g * (S + 1);
    if (!randomized) {
        for (uint32_t j = 0; j <= S; ++j) out[j] = fence(j);
        return;
    }
    rng.advance((int64_t)g * (S + 1));
    float prev = fence(0), cur = prev;                                   // lower = [t0, mids], upper = [mids, tS]
    for (uint32_t j = 0; j <= S; ++j) {
        const float next = j < S ? fence(j + 1) : cur;
        const float lower = j > 0 ? 0.5f * (cur + prev) : cur, upper = j < S ? 0.5f * (next + cur) : cur;
        out[j] = lower + (upper - lower) * rng.next_float();
        prev = cur;
        cur = next;
    }
}

// ---- hierarchical resampling (resample_along_rays :365-408 + sorted_piecewise_constant_pdf :61-117) ------------------------------------
// One warp a ray, lane l owning intervals [4l, 4l + 4).  Blur-pool, + resample_padding, the 1e-5 sum padding, the CDF with exact 0 and 1
// ends; then the S + 1 sorted u (stratified with jitter, or the linspace) are inverted by a binary search of the CDF in shared memory.
// A sample is kept inside its interval [t_k, t_k+1], so the output is sorted however the interpolation rounds.
__global__ void __launch_bounds__(32 * WARPS)
    mip_resample_kernel(uint32_t R, uint32_t S, const float* __restrict__ t_in, const float* __restrict__ w_in, float padding, int randomized,
                        Pcg32 rng, float* __restrict__ t_out) {
    __shared__ float cdf_s[WARPS][MAX_SAMPLES + 1], t_s[WARPS][MAX_SAMPLES + 1];
    const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = blockIdx.x * WARPS + warp;
    if (g >= R) return;
    const float* w = w_in + (size_t)g * S;
    const float* t = t_in + (size_t)g * (S + 1);
    float* cdf = cdf_s[warp];
    float* ts = t_s[warp];
    float wv[4], local = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t i = 4 * lane + q;
        wv[q] = 0.f;
        if (i < S) {
            const float a = w[i > 0 ? i - 1 : 0], b = w[i], c = w[i + 1 < S ? i + 1 : S - 1];
            wv[q] = 0.5f * (fmaxf(a, b) + fmaxf(b, c)) + padding;
        }
        local += wv[q];
    }
    float sum = warp_sum(local);
    const float pad = fmaxf(0.f, 1e-5f - sum);
    local = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        if (4 * lane + q < S) wv[q] += pad / S;
        local += wv[q];
    }
    sum += pad;
    // cdf[k] = min(1, sum_{i < k} pdf_i) for 0 < k < S, cdf[0] = 0, cdf[S] = 1
    float run = warp_scan(local / sum, lane) - local / sum;
    if (lane == 0) cdf[0] = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t i = 4 * lane + q;
        run += wv[q] / sum;
        if (i + 1 < S) cdf[i + 1] = fminf(1.f, run);
    }
    if (lane == 0) cdf[S] = 1.f;
    for (uint32_t j = lane; j <= S; j += 32) ts[j] = t[j];
    __syncwarp();
    if (randomized) rng.advance((int64_t)g * (S + 1) + lane);
    const float s = 1.f / (float)(S + 1);
    float* out = t_out + (size_t)g * (S + 1);
    for (uint32_t j = lane; j <= S; j += 32) {
        float u;
        if (randomized) {
            u = fminf((float)j * s + (s - EPS32) * rng.next_float(), 1.f - EPS32);
            rng.advance(31);                                             // lane's next index j + 32
        } else {
            u = (float)j * ((1.f - EPS32) / (float)S);
        }
        uint32_t lo = 0, hi = S;                                         // largest k with cdf[k] <= u: cdf[0] = 0 <= u < 1 = cdf[S]
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) / 2;
            if (cdf[mid] <= u) lo = mid;
            else hi = mid;
        }
        const float c0 = cdf[lo], c1 = cdf[lo + 1], t0 = ts[lo], t1 = ts[lo + 1];
        const float f = fminf(fmaxf((u - c0) / (c1 - c0), 0.f), 1.f);
        out[j] = fminf(fmaxf(t0 + f * (t1 - t0), t0), t1);
    }
}

// ---- fp32 encoder of the nn.Linear model: IPE (N, 48) and pos_enc(viewdir, 0, 4) (N, 27), both in the reference's column order ----------
__global__ void mip_encode_kernel(uint32_t N, uint32_t S, const float* __restrict__ rays, const float* __restrict__ t, int cylinder, int integrate,
                                  int min_deg, float* __restrict__ enc, float* __restrict__ view) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= N * 3) return;
    const uint32_t row = k / 3, dim = k % 3, ray = row / S, i = row % S;
    const float* ry = rays + (size_t)ray * RAY_FLOATS;
    const float* tt = t + (size_t)ray * (S + 1) + i;
    float mean, var;
    gaussian(ry, tt[0], tt[1], dim, cylinder, integrate, mean, var);
    float* e = enc + (size_t)row * IPE_W;
    ipe(mean, var, dim, min_deg, [&](uint32_t f, float v) { e[f] = v; });
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

// ---- composite (rays2rgb :83-96 + volumetric_rendering :278-321) ----------------------------------------------------------------------
// One warp a ray, four samples a lane.  Per sample: rgb = sigmoid(raw) (1 + 2p) - p, sigma = softplus(raw_3 + density_bias),
// sd = sigma (t_i+1 - t_i) |d|, w = (1 - e^-sd) e^-(sd of the samples before).
struct RaySamples {
    float c[4][3], sg[4][3], sd[4], dsig[4], delta[4], w[4], tb[4];   // colour, its d/draw, sd, d sigma / d raw_3, delta, weight, T before
};
template <class T>
__device__ __forceinline__ void ray_forward(const T* raw, const float* t, float dnorm, uint32_t S, float p, float bias, uint32_t lane, RaySamples& r) {
    float local = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t i = 4 * lane + q;
        r.sd[q] = 0.f;
        if (i < S) {
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const float s = 1.f / (1.f + expf(-ld(raw + (size_t)i * 4 + j)));
                r.c[q][j] = s * (1.f + 2.f * p) - p;
                r.sg[q][j] = s * (1.f - s) * (1.f + 2.f * p);
            }
            const float x = ld(raw + (size_t)i * 4 + 3) + bias;
            const float sigma = x > 20.f ? x : log1pf(expf(x));            // softplus (threshold 20, as torch / Jittor)
            r.dsig[q] = 1.f / (1.f + expf(-x));
            r.delta[q] = (t[i + 1] - t[i]) * dnorm;
            r.sd[q] = sigma * r.delta[q];
        } else {
#pragma unroll
            for (int j = 0; j < 3; ++j) r.c[q][j] = r.sg[q][j] = 0.f;
            r.dsig[q] = r.delta[q] = 0.f;
        }
        local += r.sd[q];
    }
    float before = warp_scan(local, lane) - local;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        r.tb[q] = expf(-before);
        r.w[q] = (1.f - expf(-r.sd[q])) * r.tb[q];
        before += r.sd[q];
    }
}

template <class T>
__global__ void __launch_bounds__(32 * WARPS)
    mip_composite_fwd_kernel(uint32_t R, uint32_t S, const T* __restrict__ raw, const float* __restrict__ t_in, const float* __restrict__ rays,
                             float p, float bias, int white, float* __restrict__ rgb, float* __restrict__ acc_out, float* __restrict__ dist_out,
                             float* __restrict__ w_out) {
    const uint32_t lane = threadIdx.x % 32, g = blockIdx.x * WARPS + threadIdx.x / 32;
    if (g >= R) return;
    const float* ry = rays + (size_t)g * RAY_FLOATS;
    const float* t = t_in + (size_t)g * (S + 1);
    const float dnorm = sqrtf(ry[3] * ry[3] + ry[4] * ry[4] + ry[5] * ry[5]);
    RaySamples r;
    ray_forward(raw + (size_t)g * S * 4, t, dnorm, S, p, bias, lane, r);
    float c[3] = {0.f, 0.f, 0.f}, acc = 0.f, wt = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t i = 4 * lane + q;
        if (i >= S) continue;
#pragma unroll
        for (int j = 0; j < 3; ++j) c[j] += r.w[q] * r.c[q][j];
        acc += r.w[q];
        wt += r.w[q] * (0.5f * (t[i] + t[i + 1]));
        if (w_out) w_out[(size_t)g * S + i] = r.w[q];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) c[j] = warp_sum(c[j]);
    acc = warp_sum(acc);
    wt = warp_sum(wt);
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < 3; ++j) rgb[(size_t)g * 3 + j] = white ? c[j] + (1.f - acc) : c[j];
        acc_out[g] = acc;
        // clip(distance, t_0, t_S); a ray with acc = 0 (0 / 0) gets t_0
        dist_out[g] = fminf(fmaxf(wt / acc, t[0]), t[S]);
    }
}

// Loss sum over levels of mult * sum_r mask_r |rgb_r - target_r|^2 / sum_r mask_r (runner.py:83-92; mult = coarse_loss_mult for the coarse
// level, 1 for the fine one) and its gradient with respect to every raw output, times grad_scale.  Rays [0, R) are the coarse level,
// [R, 2R) the fine one, of the same R rays.  Every block sums the mask itself, in the same order.
template <class T>
__global__ void __launch_bounds__(32 * WARPS, 1)
    mip_loss_bwd_kernel(uint32_t R, uint32_t S, const T* __restrict__ raw, const float* __restrict__ t_in, const float* __restrict__ rays,
                        const float* __restrict__ target, const float* __restrict__ mask, float p, float bias, int white, float coarse_mult,
                        float grad_scale, float* __restrict__ rgb_out, float* __restrict__ loss_out, T* __restrict__ draw) {
    __shared__ float red[32 * WARPS];
    float msum = (float)R;
    if (mask) {
        float v = 0.f;
        for (uint32_t i = threadIdx.x; i < R; i += blockDim.x) v += mask[i];
        red[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t h = blockDim.x / 2; h > 0; h >>= 1) {
            if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
            __syncthreads();
        }
        msum = red[0];
    }
    const uint32_t lane = threadIdx.x % 32, g = blockIdx.x * WARPS + threadIdx.x / 32;
    if (g >= 2 * R) return;
    const uint32_t ray = g % R;
    const float mult = g < R ? coarse_mult : 1.f, m = mask ? mask[ray] : 1.f;
    const float* ry = rays + (size_t)ray * RAY_FLOATS;
    const float* t = t_in + (size_t)g * (S + 1);
    const float dnorm = sqrtf(ry[3] * ry[3] + ry[4] * ry[4] + ry[5] * ry[5]);
    RaySamples r;
    ray_forward(raw + (size_t)g * S * 4, t, dnorm, S, p, bias, lane, r);
    float c[3] = {0.f, 0.f, 0.f}, acc = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
#pragma unroll
        for (int j = 0; j < 3; ++j) c[j] += r.w[q] * r.c[q][j];
        acc += r.w[q];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) c[j] = warp_sum(c[j]);
    acc = warp_sum(acc);
    float gr[3], loss = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if (white) c[j] += 1.f - acc;
        const float e = c[j] - target[(size_t)ray * 3 + j];
        loss += e * e;
        gr[j] = grad_scale * (mult * 2.f * m * e / msum);
        if (lane == 0) rgb_out[(size_t)g * 3 + j] = c[j];
    }
    if (lane == 0) loss_out[g] = mult * m * loss / msum;
    // dL/dsd_i = T_(i+1) gc_i - sum_(k > i) w_k gc_k with gc = dL/drgb . (colour - background of white_bkgd)
    float gc[4], local = 0.f;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        gc[q] = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j) gc[q] += gr[j] * (r.c[q][j] - (white ? 1.f : 0.f));
        local += r.w[q] * gc[q];
    }
    const float total = warp_sum(local);
    float upto = warp_scan(local, lane) - local;
    T* d = draw + (size_t)g * S * 4;
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t i = 4 * lane + q;
        if (i >= S) continue;
        upto += r.w[q] * gc[q];
        const float dsd = r.tb[q] * expf(-r.sd[q]) * gc[q] - (total - upto);
#pragma unroll
        for (int j = 0; j < 3; ++j) st(d + (size_t)i * 4 + j, r.w[q] * gr[j] * r.sg[q][j]);
        st(d + (size_t)i * 4 + 3, dsd * r.delta[q] * r.dsig[q]);
    }
}
}  // namespace mip

using namespace mip;

static inline uint32_t blocks(uint64_t n, uint32_t per) { return (uint32_t)((n + per - 1) / per); }

extern "C" {

int ngp_mip_rays(void* stream, uint32_t n, const uint32_t* pix, uint32_t W, uint32_t H, const float* c2w, float focal, float near, float far,
                 const uint8_t* images_rgba, float* rays_out, float* target_out) {
    if (n == 0) return 0;
    NGP_REQUIRE(pix && c2w && images_rgba && rays_out && target_out, "ngp_mip_rays: NULL input");
    NGP_REQUIRE(W >= 1 && H >= 3 && focal != 0.f, "ngp_mip_rays: needs W >= 1, H >= 3 and a non-zero focal length");
    mip_rays_kernel<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(n, pix, W, H, c2w, focal, near, far, images_rgba, rays_out, target_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_sample(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, int lindisp, int randomized, uint64_t rng_state,
                   uint64_t rng_inc, float* t_out) {
    NGP_REQUIRE(n_samples >= 1, "ngp_mip_sample: n_samples must be >= 1");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays && t_out, "ngp_mip_sample: NULL input");
    mip_sample_kernel<<<blocks(n_rays, 128), 128, 0, (cudaStream_t)stream>>>(n_rays, n_samples, rays, lindisp, randomized, Pcg32{rng_state, rng_inc},
                                                                            t_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_resample(void* stream, uint32_t n_rays, uint32_t n_samples, const float* t, const float* weights, float resample_padding,
                     int randomized, uint64_t rng_state, uint64_t rng_inc, float* t_out) {
    NGP_REQUIRE(n_samples >= 1 && n_samples <= MAX_SAMPLES, "ngp_mip_resample: n_samples must be in [1, 128]");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(t && weights && t_out && t != t_out, "ngp_mip_resample: NULL input, or t_out aliases t");
    mip_resample_kernel<<<blocks(n_rays, WARPS), 32 * WARPS, 0, (cudaStream_t)stream>>>(n_rays, n_samples, t, weights, resample_padding, randomized,
                                                                                       Pcg32{rng_state, rng_inc}, t_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_encode(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate, int min_deg,
                   float* enc_out, float* view_out) {
    NGP_REQUIRE(n_samples >= 1 && (uint64_t)n_rays * n_samples * 3 < (1ull << 32), "ngp_mip_encode: n_samples must be >= 1, n_rays * n_samples < 2^32 / 3");
    NGP_REQUIRE(ray_shape == 0 || ray_shape == 1, "ngp_mip_encode: ray_shape must be 0 (cone) or 1 (cylinder)");
    const uint32_t N = n_rays * n_samples;
    if (N == 0) return 0;
    NGP_REQUIRE(rays && t && enc_out && view_out, "ngp_mip_encode: NULL input");
    mip_encode_kernel<<<blocks((uint64_t)N * 3, 256), 256, 0, (cudaStream_t)stream>>>(N, n_samples, rays, t, ray_shape, integrate != 0, min_deg, enc_out,
                                                                                     view_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_composite_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, int dtype, const float* t, const float* rays,
                          float rgb_padding, float density_bias, int white_bkgd, float* rgb_out, float* acc_out, float* distance_out,
                          float* weights_out) {
    NGP_REQUIRE(n_samples >= 1 && n_samples <= MAX_SAMPLES, "ngp_mip_composite_fwd: n_samples must be in [1, 128]");
    NGP_REQUIRE(dtype == NGP_F32 || dtype == NGP_F16, "ngp_mip_composite_fwd: dtype must be NGP_F32 or NGP_F16");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(raw && t && rays && rgb_out && acc_out && distance_out, "ngp_mip_composite_fwd: NULL input");
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t b = blocks(n_rays, WARPS);
    if (dtype == NGP_F16)
        mip_composite_fwd_kernel<__half><<<b, 32 * WARPS, 0, s>>>(n_rays, n_samples, (const __half*)raw, t, rays, rgb_padding, density_bias, white_bkgd,
                                                                  rgb_out, acc_out, distance_out, weights_out);
    else
        mip_composite_fwd_kernel<float><<<b, 32 * WARPS, 0, s>>>(n_rays, n_samples, (const float*)raw, t, rays, rgb_padding, density_bias, white_bkgd,
                                                                 rgb_out, acc_out, distance_out, weights_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mip_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, int dtype, const float* t, const float* rays,
                               const float* target, const float* mask, float rgb_padding, float density_bias, int white_bkgd, float coarse_loss_mult,
                               float grad_scale, float* rgb_out, float* loss_out, void* draw_out) {
    NGP_REQUIRE(n_samples >= 1 && n_samples <= MAX_SAMPLES, "ngp_mip_composite_loss_bwd: n_samples must be in [1, 128]");
    NGP_REQUIRE(dtype == NGP_F32 || dtype == NGP_F16, "ngp_mip_composite_loss_bwd: dtype must be NGP_F32 or NGP_F16");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(raw && t && rays && target && rgb_out && loss_out && draw_out, "ngp_mip_composite_loss_bwd: NULL input");
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t b = blocks(2ull * n_rays, WARPS);
    if (dtype == NGP_F16)
        mip_loss_bwd_kernel<__half><<<b, 32 * WARPS, 0, s>>>(n_rays, n_samples, (const __half*)raw, t, rays, target, mask, rgb_padding, density_bias,
                                                             white_bkgd, coarse_loss_mult, grad_scale, rgb_out, loss_out, (__half*)draw_out);
    else
        mip_loss_bwd_kernel<float><<<b, 32 * WARPS, 0, s>>>(n_rays, n_samples, (const float*)raw, t, rays, target, mask, rgb_padding, density_bias,
                                                            white_bkgd, coarse_loss_mult, grad_scale, rgb_out, loss_out, (float*)draw_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
