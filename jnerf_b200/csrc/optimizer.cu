// N1: fused Adam + EMA + gradient zeroing in one streaming pass; N2: ray generation.
//
// The reference runs jt.nn.Adam (optims/adam.py:8-16, lr scaled by optims/expdecay.py:20-25) and then an EMA that
// overwrites the live parameters (optims/ema.py:26-37): two dense sweeps of Jittor element-wise ops over 12.2 M
// hash-grid parameters per step plus the gradient memset.  Here: one kernel, 128-bit accesses,
//   read  grad(2|4) + m(4) + v(4) + master(4)   write m(4) + v(4) + master(4) + param(2|4) [+ grad zero]
// = 30 B/param for the fp16 table -> HBM-bound (DESIGN.md).  Optimizer state is fp32; `master` is the EMA's
// `values` buffer and doubles as the fp32 master copy of fp16 parameters (documented deviation, SURVEY.md 8c).
#include "train_common.cuh"
#include "lens.cuh"
#include <cmath>
#include <cstring>

namespace {

// Each thread handles 4 consecutive parameters per slot, so that every 16-byte (fp32) / 8-byte (fp16) access of a warp is one
// fully coalesced 512 B / 256 B request; UNROLL slots are issued back to back to keep ~100 B per thread in flight.
// (The first version let a thread own 8 consecutive parameters = 32 B-strided float4 accesses: only 17 of 32 bytes per sector
//  were used per request and the kernel stalled on the LSU queue.)
template <typename PT, typename GT>
__global__ void __launch_bounds__(256) adam_ema_kernel(uint64_t n, PT* __restrict__ param, GT* __restrict__ grad, float* __restrict__ m,
                                                       float* __restrict__ v, float* __restrict__ master, AdamArgs a, int zero_grad) {
    constexpr int UNROLL = 2;
    const uint64_t n4 = n / 4, T = (uint64_t)gridDim.x * blockDim.x, g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    for (uint64_t i0 = g; i0 < n4; i0 += UNROLL * T) {
        float4 gr[UNROLL], mm[UNROLL], vv[UNROLL], ms[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const uint64_t i = i0 + u * T;
            if (i < n4) {
                if constexpr (sizeof(GT) == 2) {
                    const uint2 w = reinterpret_cast<const uint2*>(grad)[i];
                    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&w.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
                    gr[u] = make_float4(f0.x, f0.y, f1.x, f1.y);
                } else {
                    gr[u] = reinterpret_cast<const float4*>(grad)[i];
                }
                mm[u] = reinterpret_cast<const float4*>(m)[i];
                vv[u] = reinterpret_cast<const float4*>(v)[i];
                ms[u] = reinterpret_cast<const float4*>(master)[i];
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const uint64_t i = i0 + u * T;
            if (i < n4) {
                float4 p;
                p.x = adam_one(gr[u].x, mm[u].x, vv[u].x, ms[u].x, a);
                p.y = adam_one(gr[u].y, mm[u].y, vv[u].y, ms[u].y, a);
                p.z = adam_one(gr[u].z, mm[u].z, vv[u].z, ms[u].z, a);
                p.w = adam_one(gr[u].w, mm[u].w, vv[u].w, ms[u].w, a);
                reinterpret_cast<float4*>(m)[i] = mm[u];
                reinterpret_cast<float4*>(v)[i] = vv[u];
                reinterpret_cast<float4*>(master)[i] = ms[u];
                if constexpr (sizeof(PT) == 2) {
                    __half2 h0 = __floats2half2_rn(p.x, p.y), h1 = __floats2half2_rn(p.z, p.w);
                    uint2 o;
                    o.x = *reinterpret_cast<uint32_t*>(&h0);
                    o.y = *reinterpret_cast<uint32_t*>(&h1);
                    reinterpret_cast<uint2*>(param)[i] = o;
                } else {
                    reinterpret_cast<float4*>(param)[i] = p;
                }
                if (zero_grad) {
                    if constexpr (sizeof(GT) == 2) reinterpret_cast<uint2*>(grad)[i] = make_uint2(0, 0);
                    else reinterpret_cast<float4*>(grad)[i] = make_float4(0, 0, 0, 0);
                }
            }
        }
    }
    // tail (n % 4)
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const uint64_t i = n4 * 4 + threadIdx.x;
        float g1 = (float)grad[i], m1 = m[i], v1 = v[i], s1 = master[i];
        if (zero_grad) grad[i] = (GT)0.f;
        const float p = adam_one(g1, m1, v1, s1, a);
        m[i] = m1; v[i] = v1; master[i] = s1; param[i] = (PT)p;
    }
}

// The training step's whole optimizer tail in one launch, after ngp_network_bwd_fx.  It computes exactly what the backward's slot
// reduction and fixed-point flush (ngp_network_bwd) followed by adam_ema_kernel on the three gradients compute, without the fp16
// table gradient in between: per table parameter 8 + 26 bytes plus 8 for every touched one, against 8 + 12 f + 30 for that sequence.
//  * blocks [0, SWEEP_W_BLOCKS), scheduled first: one MLP weight each thread -- the sum of the backward's per-CTA slots in CTA order,
//    formed as wgrad_reduce_kernel forms it and added to a zero gradient, then Adam+EMA;
//  * the other blocks stream the hash table, one entry (2 parameters) per slot: the fixed-point sums rounded once to fp16, as the
//    flush rounds them into a zeroed gradient, nonzero scratch entries cleared for the next backward, then Adam+EMA.
constexpr uint32_t SWEEP_THREADS = 256, SWEEP_W_BLOCKS = (W_PART + SWEEP_THREADS - 1) / SWEEP_THREADS;
struct SweepTensor { __half* param; float *m, *v, *master; };

// the gradient of one table entry, as the flush leaves it in a zeroed fp16 gradient (the product is exact: FX_INV is a power of two)
__device__ __forceinline__ float2 fx_grad(longlong2 q) {
    if (!(q.x | q.y)) return make_float2(0.f, 0.f);
    return __half22float2(__floats2half2_rn(__fmul_rn(__ll2float_rn(q.x), FX_INV), __fmul_rn(__ll2float_rn(q.y), FX_INV)));
}

__global__ void __launch_bounds__(SWEEP_THREADS) train_sweep_kernel(uint64_t n_entries, SweepTensor tab, longlong2* __restrict__ fx,
                                                                    const float* __restrict__ part, uint32_t nparts, SweepTensor wd, SweepTensor wr,
                                                                    AdamArgs a) {
    if (blockIdx.x < SWEEP_W_BLOCKS) {
        const uint32_t e = blockIdx.x * SWEEP_THREADS + threadIdx.x;
        if (e >= (uint32_t)W_PART) return;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        uint32_t k = 0;
#pragma unroll 4
        for (; k + 4 <= nparts; k += 4) {
            a0 += part[(size_t)k * W_PART + e];
            a1 += part[(size_t)(k + 1) * W_PART + e];
            a2 += part[(size_t)(k + 2) * W_PART + e];
            a3 += part[(size_t)(k + 3) * W_PART + e];
        }
        for (; k < nparts; ++k) a0 += part[(size_t)k * W_PART + e];
        const float g = __fadd_rn(0.f, (a0 + a1) + (a2 + a3));
        const bool d = e < (uint32_t)WD_N;
        const uint32_t j = d ? e : e - WD_N;
        float* wm = (d ? wd.m : wr.m) + j;
        float* wv = (d ? wd.v : wr.v) + j;
        float* ws = (d ? wd.master : wr.master) + j;
        float m1 = *wm, v1 = *wv, s1 = *ws;
        const float p = adam_one(g, m1, v1, s1, a);
        *wm = m1; *wv = v1; *ws = s1;
        (d ? wd.param : wr.param)[j] = __float2half_rn(p);
        return;
    }
    // one entry (2 parameters) per thread and slot: every access of a warp -- 16 B of scratch, 8 B of m / v / master, 4 B of
    // parameters per lane -- is one contiguous request whose sectors are used whole
    constexpr int UNROLL = 4;
    const uint64_t T = (uint64_t)(gridDim.x - SWEEP_W_BLOCKS) * SWEEP_THREADS;
    const uint64_t g0 = (uint64_t)(blockIdx.x - SWEEP_W_BLOCKS) * SWEEP_THREADS + threadIdx.x;
    for (uint64_t i0 = g0; i0 < n_entries; i0 += UNROLL * T) {
        longlong2 q[UNROLL];
        float2 mm[UNROLL], vv[UNROLL], ms[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const uint64_t i = i0 + u * T;
            if (i < n_entries) {
                q[u] = fx[i];
                mm[u] = reinterpret_cast<const float2*>(tab.m)[i];
                vv[u] = reinterpret_cast<const float2*>(tab.v)[i];
                ms[u] = reinterpret_cast<const float2*>(tab.master)[i];
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const uint64_t i = i0 + u * T;
            if (i < n_entries) {
                const float2 g = fx_grad(q[u]);
                if (q[u].x | q[u].y) fx[i] = make_longlong2(0, 0);
                const float px = adam_one(g.x, mm[u].x, vv[u].x, ms[u].x, a);
                const float py = adam_one(g.y, mm[u].y, vv[u].y, ms[u].y, a);
                reinterpret_cast<float2*>(tab.m)[i] = mm[u];
                reinterpret_cast<float2*>(tab.v)[i] = vv[u];
                reinterpret_cast<float2*>(tab.master)[i] = ms[u];
                reinterpret_cast<__half2*>(tab.param)[i] = __floats2half2_rn(px, py);
            }
        }
    }
}

// LENS: the pixel's normalised coordinate is undistorted through image id's (k1, k2, p1, p2) = lens[id] first (lens.cuh); without it,
// a pinhole ray, as the reference builds every ray.
template <bool LENS>
__global__ void raygen_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t W, uint32_t H, const float* __restrict__ xforms,
                              const float* __restrict__ focal, const float* __restrict__ principal, uint32_t* __restrict__ img_id,
                              float* __restrict__ rays_o, float* __restrict__ rays_d, const float4* __restrict__ lens) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = pix[i] / (H * W), off = pix[i] % (H * W);                  // dataset.py:173-174
    const float* m = xforms + 12 * (size_t)id;                                     // column-major 3x4
    const float x = ((off % W) + 0.5f) / W, y = ((off / W) + 0.5f) / H;            // :180-181
    float dx = (x - principal[2 * id]) * W / focal[2 * id], dy = (y - principal[2 * id + 1]) * H / focal[2 * id + 1];
    if constexpr (LENS) lens_undistort(dx, dy, lens[id]);
    const float d0 = m[0] * dx + m[3] * dy + m[6], d1 = m[1] * dx + m[4] * dy + m[7], d2 = m[2] * dx + m[5] * dy + m[8];
    const float nrm = fmaxf(sqrtf(d0 * d0 + d1 * d1 + d2 * d2), 1e-12f);           // jt.normalize
    img_id[i] = id;
    rays_o[3 * (size_t)i] = m[9]; rays_o[3 * (size_t)i + 1] = m[10]; rays_o[3 * (size_t)i + 2] = m[11];
    rays_d[3 * (size_t)i] = d0 / nrm; rays_d[3 * (size_t)i + 1] = d1 / nrm; rays_d[3 * (size_t)i + 2] = d2 / nrm;
}

// N2 fused: ray generation + RGBA gather + target = rgb*a + bg*(1-a)  (dataset.py:172-188, runner.py:66-68) in one launch.
// LENS as in raygen_kernel: the same rays, bit for bit; the target lookup and blend do not depend on it.
template <typename IMG, bool LENS>
__global__ void prepare_batch_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t W, uint32_t H, const float* __restrict__ xforms,
                                     const float* __restrict__ focal, const float* __restrict__ principal, const IMG* __restrict__ images,
                                     const float* __restrict__ bg, uint32_t* __restrict__ img_id, float* __restrict__ rays_o,
                                     float* __restrict__ rays_d, float* __restrict__ target, const float4* __restrict__ lens) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t px = pix[i];
    const uint32_t id = px / (H * W), off = px % (H * W);
    const float* m = xforms + 12 * (size_t)id;
    const float x = ((off % W) + 0.5f) / W, y = ((off / W) + 0.5f) / H;
    float dx = (x - principal[2 * id]) * W / focal[2 * id], dy = (y - principal[2 * id + 1]) * H / focal[2 * id + 1];
    if constexpr (LENS) lens_undistort(dx, dy, lens[id]);
    const float d0 = m[0] * dx + m[3] * dy + m[6], d1 = m[1] * dx + m[4] * dy + m[7], d2 = m[2] * dx + m[5] * dy + m[8];
    const float nrm = fmaxf(sqrtf(d0 * d0 + d1 * d1 + d2 * d2), 1e-12f);
    img_id[i] = id;
    rays_o[3 * (size_t)i] = m[9]; rays_o[3 * (size_t)i + 1] = m[10]; rays_o[3 * (size_t)i + 2] = m[11];
    rays_d[3 * (size_t)i] = d0 / nrm; rays_d[3 * (size_t)i + 1] = d1 / nrm; rays_d[3 * (size_t)i + 2] = d2 / nrm;
    float4 c;
    if constexpr (sizeof(IMG) == 1) {
        const uchar4 u = reinterpret_cast<const uchar4*>(images)[px];
        c = make_float4(u.x / 255.0f, u.y / 255.0f, u.z / 255.0f, u.w / 255.0f);      // read_image: uint8 / 255
    } else {
        c = reinterpret_cast<const float4*>(images)[px];
    }
    const float ia = 1.0f - c.w;
    target[3 * (size_t)i] = c.x * c.w + bg[3 * (size_t)i] * ia;
    target[3 * (size_t)i + 1] = c.y * c.w + bg[3 * (size_t)i + 1] * ia;
    target[3 * (size_t)i + 2] = c.z * c.w + bg[3 * (size_t)i + 2] * ia;
}

// Captures whose frames carry their own cameras (plugin/dataset.py, per_frame_cameras): image i owns the global pixel ids
// [offsets[i], offsets[i+1]) of a ragged, row-major table, and is wh[i] = (w, h) pixels.  The image of pixel p is found by a binary
// search over the n_images + 1 prefix sums; off = p - offsets[id] is then the pixel's row-major offset in its own image.
__device__ __forceinline__ uint32_t frame_of_pixel(uint32_t p, uint32_t n_images, const uint32_t* __restrict__ offsets) {
    uint32_t lo = 0, hi = n_images;                        // offsets[lo] <= p < offsets[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(offsets + mid) <= p) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The ray of raygen_kernel<LENS> for the pixel p of a ragged capture, with the image's own W and H: the same operations in the same
// order, so a capture whose images all share one size gives raygen_kernel's rays bit for bit.
template <bool LENS>
__device__ __forceinline__ uint32_t frame_ray(uint32_t p, uint32_t n_images, const uint32_t* __restrict__ offsets, const uint2* __restrict__ wh,
                                              const float* __restrict__ xforms, const float* __restrict__ focal,
                                              const float* __restrict__ principal, const float4* __restrict__ lens, uint32_t i,
                                              float* __restrict__ rays_o, float* __restrict__ rays_d) {
    const uint32_t id = frame_of_pixel(p, n_images, offsets);
    const uint2 s = __ldg(wh + id);
    const uint32_t W = s.x, H = s.y, off = p - __ldg(offsets + id);
    const float* m = xforms + 12 * (size_t)id;
    const float x = ((off % W) + 0.5f) / W, y = ((off / W) + 0.5f) / H;
    float dx = (x - principal[2 * id]) * W / focal[2 * id], dy = (y - principal[2 * id + 1]) * H / focal[2 * id + 1];
    if constexpr (LENS) lens_undistort(dx, dy, lens[id]);
    const float d0 = m[0] * dx + m[3] * dy + m[6], d1 = m[1] * dx + m[4] * dy + m[7], d2 = m[2] * dx + m[5] * dy + m[8];
    const float nrm = fmaxf(sqrtf(d0 * d0 + d1 * d1 + d2 * d2), 1e-12f);
    rays_o[3 * (size_t)i] = m[9]; rays_o[3 * (size_t)i + 1] = m[10]; rays_o[3 * (size_t)i + 2] = m[11];
    rays_d[3 * (size_t)i] = d0 / nrm; rays_d[3 * (size_t)i + 1] = d1 / nrm; rays_d[3 * (size_t)i + 2] = d2 / nrm;
    return id;
}

template <bool LENS>
__global__ void raygen_cams_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t n_images, const uint32_t* __restrict__ offsets,
                                   const uint2* __restrict__ wh, const float* __restrict__ xforms, const float* __restrict__ focal,
                                   const float* __restrict__ principal, const float4* __restrict__ lens, uint32_t* __restrict__ img_id,
                                   float* __restrict__ rays_o, float* __restrict__ rays_d) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    img_id[i] = frame_ray<LENS>(pix[i], n_images, offsets, wh, xforms, focal, principal, lens, i, rays_o, rays_d);
}

// raygen_cams_kernel + the pixel's RGBA from the ragged (total_pixels, 4) table, blended as prepare_batch_kernel blends it
template <typename IMG, bool LENS>
__global__ void prepare_batch_cams_kernel(uint32_t n, const uint32_t* __restrict__ pix, uint32_t n_images, const uint32_t* __restrict__ offsets,
                                          const uint2* __restrict__ wh, const float* __restrict__ xforms, const float* __restrict__ focal,
                                          const float* __restrict__ principal, const float4* __restrict__ lens, const IMG* __restrict__ images,
                                          const float* __restrict__ bg, uint32_t* __restrict__ img_id, float* __restrict__ rays_o,
                                          float* __restrict__ rays_d, float* __restrict__ target) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t px = pix[i];
    img_id[i] = frame_ray<LENS>(px, n_images, offsets, wh, xforms, focal, principal, lens, i, rays_o, rays_d);
    float4 c;
    if constexpr (sizeof(IMG) == 1) {
        const uchar4 u = reinterpret_cast<const uchar4*>(images)[px];
        c = make_float4(u.x / 255.0f, u.y / 255.0f, u.z / 255.0f, u.w / 255.0f);
    } else {
        c = reinterpret_cast<const float4*>(images)[px];
    }
    const float ia = 1.0f - c.w;
    target[3 * (size_t)i] = c.x * c.w + bg[3 * (size_t)i] * ia;
    target[3 * (size_t)i + 1] = c.y * c.w + bg[3 * (size_t)i + 1] * ia;
    target[3 * (size_t)i + 2] = c.z * c.w + bg[3 * (size_t)i + 2] * ia;
}

// target = rgb*a + bg*(1-a) (runner.py:68) for a ray batch that arrives with its RGBA already gathered (host-fed batches)
__global__ void blend_target_kernel(uint32_t n, const float4* __restrict__ rgba, const float* __restrict__ bg, float* __restrict__ target) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 c = rgba[i];
    const float ia = 1.0f - c.w;
    target[3 * (size_t)i] = c.x * c.w + bg[3 * (size_t)i] * ia;
    target[3 * (size_t)i + 1] = c.y * c.w + bg[3 * (size_t)i + 1] * ia;
    target[3 * (size_t)i + 2] = c.z * c.w + bg[3 * (size_t)i + 2] * ia;
}

// ---------------------------------------------------------------------------------------------------------------------
// 8e: data-parallel gradient exchange + optimizer in ONE kernel over NVLink peer memory.
//
// Every rank maps every other rank's gradient buffers, parameter table and flag block (CUDA IPC, dp.py).  Rank k owns the
// slice [k*slice_len, (k+1)*slice_len) of the padded hash table:
//   1. block 0 tells every peer "my gradients of this step are complete" (release store of `epoch` into the peer's flag block;
//      the kernel is stream-ordered behind the backward kernel), then every block waits until all peers have said so;
//   2. reduce-scatter by pulling: g = sum over ranks of table_grad[r][slice] (128-bit loads over NVLink), fused Adam + EMA
//      on the slice (optimizer state exists only for the slice: 1/W of the 171 MB state traffic per GPU);
//   3. all-gather by pushing: the updated fp16 slice is stored into every rank's table (128-bit stores over NVLink);
//   4. the two small MLP weight tensors (10 240 values) are all-reduced by every rank reading every rank's copy -- same order
//      of summation everywhere, so the replicas stay bit-identical -- and updated locally;
//   5. the last block to finish tells every peer "my stores into your table are complete and I no longer read your
//      gradients"; ngp_dp_exchange_wait() consumes those flags before the next forward pass / gradient zeroing.
// Replaces reduce-scatter + all-reduce + 3 Adam launches + all-gather (NCCL path, dp.py) with one launch.
constexpr int DP_MAX_WORLD = 16;
constexpr int DP_FLAG_GRADS = 0, DP_FLAG_DONE = 16, DP_FLAG_COUNTER = 32, DP_FLAG_WORDS = 64;

struct DpPeers {
    __half* table[DP_MAX_WORLD];
    __half* table_grad[DP_MAX_WORLD];
    float* w_grad[DP_MAX_WORLD];
    uint32_t* flags[DP_MAX_WORLD];
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Bounded spin (a dead peer must not hang the GPU): traps after 20 s.
__device__ __forceinline__ void wait_flag(const uint32_t* p, uint32_t epoch) {
    const uint64_t t0 = global_timer_ns();
#pragma unroll 1
    while ((int32_t)(ld_acquire_sys(p) - epoch) < 0) {
        if (global_timer_ns() - t0 > 20ull * 1000000000ull) __trap();
    }
}

__global__ void __launch_bounds__(256, 2) dp_exchange_kernel(DpPeers P, int W, int rank, uint64_t slice_len, uint32_t n_w, uint32_t epoch,
                                                          float* m, float* v, float* master, __half* w_param, float* w_m, float* w_v,
                                                          float* w_master, AdamArgs a) {
    if (blockIdx.x == 0 && threadIdx.x < W) {
        __threadfence_system();
        st_release_sys(P.flags[threadIdx.x] + DP_FLAG_GRADS + rank, epoch);
    }
    if (threadIdx.x < W) wait_flag(P.flags[rank] + DP_FLAG_GRADS + threadIdx.x, epoch);
    __syncthreads();

    const uint64_t lo = (uint64_t)rank * slice_len, n8 = slice_len / 8;
    const uint64_t T = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n8; i += T) {
        float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        uint4 w[DP_MAX_WORLD];
#pragma unroll
        for (int r = 0; r < DP_MAX_WORLD; ++r)
            if (r < W) w[r] = *reinterpret_cast<uint4*>(P.table_grad[r] + lo + 8 * i);       // W independent 16 B loads in flight
        float4 mm[2], vv[2], ms[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mm[h] = reinterpret_cast<const float4*>(m)[2 * i + h];
            vv[h] = reinterpret_cast<const float4*>(v)[2 * i + h];
            ms[h] = reinterpret_cast<const float4*>(master)[2 * i + h];
        }
#pragma unroll
        for (int r = 0; r < DP_MAX_WORLD; ++r) {
            if (r < W) {
                const uint32_t u[4] = {w[r].x, w[r].y, w[r].z, w[r].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u[k]));
                    g[2 * k] += f.x;
                    g[2 * k + 1] += f.y;
                }
            }
        }
        float p[8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            p[4 * h + 0] = adam_one(g[4 * h + 0], mm[h].x, vv[h].x, ms[h].x, a);
            p[4 * h + 1] = adam_one(g[4 * h + 1], mm[h].y, vv[h].y, ms[h].y, a);
            p[4 * h + 2] = adam_one(g[4 * h + 2], mm[h].z, vv[h].z, ms[h].z, a);
            p[4 * h + 3] = adam_one(g[4 * h + 3], mm[h].w, vv[h].w, ms[h].w, a);
            reinterpret_cast<float4*>(m)[2 * i + h] = mm[h];
            reinterpret_cast<float4*>(v)[2 * i + h] = vv[h];
            reinterpret_cast<float4*>(master)[2 * i + h] = ms[h];
        }
        uint4 o;
        {
            __half2 h0 = __floats2half2_rn(p[0], p[1]), h1 = __floats2half2_rn(p[2], p[3]), h2 = __floats2half2_rn(p[4], p[5]),
                    h3 = __floats2half2_rn(p[6], p[7]);
            o.x = *reinterpret_cast<uint32_t*>(&h0);
            o.y = *reinterpret_cast<uint32_t*>(&h1);
            o.z = *reinterpret_cast<uint32_t*>(&h2);
            o.w = *reinterpret_cast<uint32_t*>(&h3);
        }
#pragma unroll
        for (int r = 0; r < DP_MAX_WORLD; ++r)
            if (r < W) *reinterpret_cast<uint4*>(P.table[r] + lo + 8 * i) = o;
    }
    // MLP weights: identical all-reduce + update on every rank
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_w; j += (uint32_t)T) {
        float g = 0.f;
        for (int r = 0; r < W; ++r) g += P.w_grad[r][j];
        float m1 = w_m[j], v1 = w_v[j], s1 = w_master[j];
        const float p = adam_one(g, m1, v1, s1, a);
        w_m[j] = m1; w_v[j] = v1; w_master[j] = s1;
        w_param[j] = __float2half_rn(p);
    }
    // completion: all of this rank's peer stores are performed before any peer sees the flag
    __threadfence_system();
    __syncthreads();
    __shared__ bool last;
    uint32_t* mine = P.flags[rank];
    if (threadIdx.x == 0) last = atomicAdd(mine + DP_FLAG_COUNTER, 1u) == gridDim.x - 1;
    __syncthreads();
    if (last) {
        __threadfence();
        if (threadIdx.x < W) st_release_sys(P.flags[threadIdx.x] + DP_FLAG_DONE + rank, epoch);
        if (threadIdx.x == 0) mine[DP_FLAG_COUNTER] = 0;
    }
}

__global__ void dp_wait_kernel(const uint32_t* my_flags, int W, uint32_t epoch) {
    if (threadIdx.x < W) wait_flag(my_flags + DP_FLAG_DONE + threadIdx.x, epoch);
}

template <bool LENS>
void launch_prepare_batch(cudaStream_t s, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms,
                                 const float* focal, const float* principal, const void* images_rgba, int image_is_u8, const float* bg,
                                 uint32_t* img_id_out, float* rays_o, float* rays_d, float* target, const float4* lens) {
    if (image_is_u8) prepare_batch_kernel<uint8_t, LENS><<<(n + 127) / 128, 128, 0, s>>>(n, pix_index, W, H, xforms, focal, principal, (const uint8_t*)images_rgba, bg, img_id_out, rays_o, rays_d, target, lens);
    else prepare_batch_kernel<float, LENS><<<(n + 127) / 128, 128, 0, s>>>(n, pix_index, W, H, xforms, focal, principal, (const float*)images_rgba, bg, img_id_out, rays_o, rays_d, target, lens);
}

template <bool LENS>
void launch_prepare_batch_cams(cudaStream_t s, uint32_t n, const uint32_t* pix_index, uint32_t n_images, const uint32_t* offsets, const uint2* wh,
                               const float* xforms, const float* focal, const float* principal, const float4* lens, const void* images_rgba,
                               int image_is_u8, const float* bg, uint32_t* img_id_out, float* rays_o, float* rays_d, float* target) {
    if (image_is_u8) prepare_batch_cams_kernel<uint8_t, LENS><<<(n + 127) / 128, 128, 0, s>>>(n, pix_index, n_images, offsets, wh, xforms, focal, principal, lens, (const uint8_t*)images_rgba, bg, img_id_out, rays_o, rays_d, target);
    else prepare_batch_cams_kernel<float, LENS><<<(n + 127) / 128, 128, 0, s>>>(n, pix_index, n_images, offsets, wh, xforms, focal, principal, lens, (const float*)images_rgba, bg, img_id_out, rays_o, rays_d, target);
}

}  // namespace

extern "C" {

static AdamArgs make_adam_args(float lr, float beta1, float beta2, float eps, uint32_t step, float ema_decay, float grad_scale) {
    AdamArgs a;
    const double n1 = 1.0 - std::pow((double)beta1, (double)step), n2 = 1.0 - std::pow((double)beta2, (double)step);
    a.step_size = (float)(lr * std::sqrt(n2) / n1);
    a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.decay = ema_decay; a.grad_scale = grad_scale;
    a.debias_old = (float)(1.0 - std::pow((double)ema_decay, (double)step - 1.0));
    a.debias_new = (float)(1.0 / (1.0 - std::pow((double)ema_decay, (double)step)));
    return a;
}

int ngp_adam_ema(void* stream, uint64_t n, void* param, int param_dtype, void* grad, int grad_dtype, float grad_scale, float* m, float* v,
                 float* master, float lr, float beta1, float beta2, float eps, uint32_t step, float ema_decay, int zero_grad) {
    NGP_REQUIRE(step >= 1, "ngp_adam_ema: step is 1-based");
    if (n == 0) return 0;
    const AdamArgs a = make_adam_args(lr, beta1, beta2, eps, step, ema_decay, grad_scale);
    cudaStream_t s = (cudaStream_t)stream;
    const uint64_t n4 = (n + 3) / 4;
    const uint32_t blocks = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n4 + 511) / 512, (uint64_t)ngp_num_sms() * 32));
    if (param_dtype == 1 && grad_dtype == 1) adam_ema_kernel<__half, __half><<<blocks, 256, 0, s>>>(n, (__half*)param, (__half*)grad, m, v, master, a, zero_grad);
    else if (param_dtype == 1 && grad_dtype == 0) adam_ema_kernel<__half, float><<<blocks, 256, 0, s>>>(n, (__half*)param, (float*)grad, m, v, master, a, zero_grad);
    else if (param_dtype == 0 && grad_dtype == 0) adam_ema_kernel<float, float><<<blocks, 256, 0, s>>>(n, (float*)param, (float*)grad, m, v, master, a, zero_grad);
    else NGP_REQUIRE(false, "ngp_adam_ema: unsupported dtype combination");
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_train_sweep(void* stream, uint64_t n_entries, void* table, float* m, float* v, float* master, void* fx, const float* w_part,
                    uint32_t bwd_rows, void* w_density, float* wd_m, float* wd_v, float* wd_master, void* w_rgb, float* wr_m, float* wr_v,
                    float* wr_master, float lr, float beta1, float beta2, float eps, uint32_t step, float ema_decay) {
    NGP_REQUIRE(step >= 1, "ngp_train_sweep: step is 1-based");
    NGP_REQUIRE(fx != nullptr && w_part != nullptr, "ngp_train_sweep: the backward's fixed-point scratch and weight-gradient slots are required");
    const uint32_t blocks = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n_entries + 4 * SWEEP_THREADS - 1) / (4 * SWEEP_THREADS),
                                                                           (uint64_t)ngp_num_sms() * 32));
    train_sweep_kernel<<<SWEEP_W_BLOCKS + blocks, SWEEP_THREADS, 0, (cudaStream_t)stream>>>(
        n_entries, SweepTensor{(__half*)table, m, v, master}, (longlong2*)fx, w_part, bwd_ctas(bwd_rows),
        SweepTensor{(__half*)w_density, wd_m, wd_v, wd_master}, SweepTensor{(__half*)w_rgb, wr_m, wr_v, wr_master},
        make_adam_args(lr, beta1, beta2, eps, step, ema_decay, 1.0f));
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_dp_exchange_step(void* stream, int world, int rank, uint64_t slice_len, uint32_t n_w, void* const* peer_table,
                         void* const* peer_table_grad, float* const* peer_w_grad, uint32_t* const* peer_flags, uint32_t epoch, float* m,
                         float* v, float* master, void* w_param, float* w_m, float* w_v, float* w_master, float grad_scale, float lr,
                         float beta1, float beta2, float eps, uint32_t step, float ema_decay) {
    NGP_REQUIRE(world >= 1 && world <= DP_MAX_WORLD && rank >= 0 && rank < world, "ngp_dp_exchange_step: world must be 1..16 and rank < world");
    NGP_REQUIRE(slice_len % 256 == 0, "ngp_dp_exchange_step: slice_len must be a multiple of 256 (dp.padded_len)");
    NGP_REQUIRE(step >= 1 && epoch >= 1, "ngp_dp_exchange_step: step and epoch are 1-based");
    DpPeers P;
    for (int r = 0; r < DP_MAX_WORLD; ++r) {
        const int q = r < world ? r : rank;
        P.table[r] = (__half*)peer_table[q];
        P.table_grad[r] = (__half*)peer_table_grad[q];
        P.w_grad[r] = peer_w_grad[q];
        P.flags[r] = peer_flags[q];
    }
    const AdamArgs a = make_adam_args(lr, beta1, beta2, eps, step, ema_decay, grad_scale);
    // every block spins on peer flags before it starts: keep the grid co-resident (2 CTAs/SM, enforced by __launch_bounds__)
    const uint64_t n8 = slice_len / 8;
    const uint32_t blocks = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n8 + 255) / 256, (uint64_t)ngp_num_sms() * 2));
    dp_exchange_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(P, world, rank, slice_len, n_w, epoch, m, v, master, (__half*)w_param, w_m, w_v,
                                                                 w_master, a);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_dp_exchange_wait(void* stream, int world, const uint32_t* my_flags, uint32_t epoch) {
    NGP_REQUIRE(world >= 1 && world <= DP_MAX_WORLD, "ngp_dp_exchange_wait: world must be 1..16");
    dp_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(my_flags, world, epoch);
    NGP_LAUNCH_CHECK();
    return 0;
}

// CUDA IPC plumbing for the peer mapping (runtime API only; the base of the allocation comes from the driver entry point so that
// the library keeps no link-time dependency on libcuda and still loads on a machine without a GPU).
int ngp_ipc_export(const void* dev_ptr, uint8_t* handle64, uint64_t* offset) {
    typedef int (*GetRange)(unsigned long long*, size_t*, unsigned long long);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    NGP_CHECK_CUDA(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qr));
    NGP_REQUIRE(fn != nullptr && qr == cudaDriverEntryPointSuccess, "ngp_ipc_export: cuMemGetAddressRange not available");
    unsigned long long base = 0;
    size_t size = 0;
    NGP_REQUIRE(((GetRange)fn)(&base, &size, (unsigned long long)(uintptr_t)dev_ptr) == 0, "ngp_ipc_export: not a device allocation");
    cudaIpcMemHandle_t h;
    NGP_CHECK_CUDA(cudaIpcGetMemHandle(&h, (void*)(uintptr_t)base));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64, &h, 64);
    *offset = (uint64_t)((uintptr_t)dev_ptr - (uintptr_t)base);
    return 0;
}

int ngp_ipc_open(const uint8_t* handle64, uint64_t offset, void** dev_ptr) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void* base = nullptr;
    NGP_CHECK_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    *dev_ptr = (void*)((uintptr_t)base + offset);
    return 0;
}

int ngp_ipc_close(void* dev_ptr, uint64_t offset) {
    NGP_CHECK_CUDA(cudaIpcCloseMemHandle((void*)((uintptr_t)dev_ptr - offset)));
    return 0;
}

int ngp_prepare_batch(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms, const float* focal,
                      const float* principal, const void* images_rgba, int image_is_u8, const float* bg, uint32_t* img_id_out, float* rays_o,
                      float* rays_d, float* target) {
    if (n == 0) return 0;
    launch_prepare_batch<false>((cudaStream_t)stream, n, pix_index, W, H, xforms, focal, principal, images_rgba, image_is_u8, bg, img_id_out, rays_o,
                                rays_d, target, nullptr);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_prepare_batch_lens(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms, const float* focal,
                           const float* principal, const float* distortion, const void* images_rgba, int image_is_u8, const float* bg,
                           uint32_t* img_id_out, float* rays_o, float* rays_d, float* target) {
    if (n == 0) return 0;
    NGP_REQUIRE(distortion != nullptr && (reinterpret_cast<uintptr_t>(distortion) & 15) == 0,
                "ngp_prepare_batch_lens: distortion must be a 16-byte aligned (n_images, 4) float array");
    launch_prepare_batch<true>((cudaStream_t)stream, n, pix_index, W, H, xforms, focal, principal, images_rgba, image_is_u8, bg, img_id_out, rays_o,
                               rays_d, target, reinterpret_cast<const float4*>(distortion));
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_blend_target(void* stream, uint32_t n, const float* rgba, const float* bg, float* target) {
    if (n == 0) return 0;
    blend_target_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, reinterpret_cast<const float4*>(rgba), bg, target);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_raygen(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms, const float* focal,
               const float* principal, uint32_t* img_id_out, float* rays_o, float* rays_d) {
    if (n == 0) return 0;
    raygen_kernel<false><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, pix_index, W, H, xforms, focal, principal, img_id_out, rays_o, rays_d,
                                                                            nullptr);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_raygen_lens(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms, const float* focal,
                    const float* principal, const float* distortion, uint32_t* img_id_out, float* rays_o, float* rays_d) {
    if (n == 0) return 0;
    NGP_REQUIRE(distortion != nullptr && (reinterpret_cast<uintptr_t>(distortion) & 15) == 0,
                "ngp_raygen_lens: distortion must be a 16-byte aligned (n_images, 4) float array");
    raygen_kernel<true><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, pix_index, W, H, xforms, focal, principal, img_id_out, rays_o, rays_d,
                                                                           reinterpret_cast<const float4*>(distortion));
    NGP_LAUNCH_CHECK();
    return 0;
}

static int require_cams(const char* fn, uint32_t n_images, const uint32_t* pixel_offsets, const uint32_t* wh, const float* distortion) {
    NGP_REQUIRE(n_images >= 1 && pixel_offsets != nullptr, std::string(fn) + ": needs n_images >= 1 and the (n_images + 1) pixel offsets");
    NGP_REQUIRE(wh != nullptr && (reinterpret_cast<uintptr_t>(wh) & 7) == 0, std::string(fn) + ": wh must be an 8-byte aligned (n_images, 2) uint32 array");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(distortion) & 15) == 0, std::string(fn) + ": distortion must be NULL or a 16-byte aligned (n_images, 4) float array");
    return 0;
}

int ngp_raygen_cams(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t n_images, const uint32_t* pixel_offsets, const uint32_t* wh,
                    const float* xforms, const float* focal, const float* principal, const float* distortion, uint32_t* img_id_out, float* rays_o,
                    float* rays_d) {
    if (n == 0) return 0;
    if (const int e = require_cams("ngp_raygen_cams", n_images, pixel_offsets, wh, distortion)) return e;
    const uint2* wh2 = reinterpret_cast<const uint2*>(wh);
    const float4* lens = reinterpret_cast<const float4*>(distortion);
    if (lens) raygen_cams_kernel<true><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, pix_index, n_images, pixel_offsets, wh2, xforms, focal, principal, lens, img_id_out, rays_o, rays_d);
    else raygen_cams_kernel<false><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, pix_index, n_images, pixel_offsets, wh2, xforms, focal, principal, nullptr, img_id_out, rays_o, rays_d);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_prepare_batch_cams(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t n_images, const uint32_t* pixel_offsets, const uint32_t* wh,
                           const float* xforms, const float* focal, const float* principal, const float* distortion, const void* images_rgba,
                           int image_is_u8, const float* bg, uint32_t* img_id_out, float* rays_o, float* rays_d, float* target) {
    if (n == 0) return 0;
    if (const int e = require_cams("ngp_prepare_batch_cams", n_images, pixel_offsets, wh, distortion)) return e;
    const uint2* wh2 = reinterpret_cast<const uint2*>(wh);
    const float4* lens = reinterpret_cast<const float4*>(distortion);
    cudaStream_t s = (cudaStream_t)stream;
    if (lens) launch_prepare_batch_cams<true>(s, n, pix_index, n_images, pixel_offsets, wh2, xforms, focal, principal, lens, images_rgba, image_is_u8, bg, img_id_out, rays_o, rays_d, target);
    else launch_prepare_batch_cams<false>(s, n, pix_index, n_images, pixel_offsets, wh2, xforms, focal, principal, nullptr, images_rgba, image_is_u8, bg, img_id_out, rays_o, rays_d, target);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
