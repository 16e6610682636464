// Whole-frame renderer: a wavefront loop over rounds that stops a ray once it is opaque (DESIGN.md section 4, "Rendering").
// Compiled with -fmad=false like sampler.cu: the march takes the step rule of march_common.cuh, so every ray visits the samples that
// ngp_march produces for it, bit for bit, in order.
//
// What it stands in for: runner.py:197-264 tiles a frame into n_rays_per_batch batches, marches every sample of every ray
// (ray_sampler.h) and composites all of them (calc_rgb.h:151-212, no early stop).  Here one call covers any number of rays:
//   init            slab test, near distance and jitter per ray; rays that miss the box finish at once; compaction -> alive list
//   march round     each alive ray continues its march from its saved (t, steps taken) for up to K more samples; per-ray counts ->
//                   block sums -> one-CTA scan of the block sums -> dense NerfCoordinate rows in alive-list (= ray) order
//   (network)       the caller runs the fused forward (ngp_network_fwd) over the round's rows, bounded by the device row count
//   composite round each alive ray composites its rows one after another; it stops after the first sample that brings T below
//                   min_transmittance, or when its march has ended; the others form the next round's alive list (order-preserving
//                   compaction).  The alive count is read back: 4 bytes a round.
// The result does not depend on K or on the row capacity: the march resumes exactly where it stopped and the stopping rule is
// applied sample by sample.  No float atomics anywhere: every scan is a fixed-order block scan.
#include "march_common.cuh"

namespace {

constexpr uint32_t RB = 256;                    // threads per block of the per-ray kernels (one thread per ray / alive entry)

// Exclusive scan of v over the block; *total = the block's sum.  Once per kernel (static shared memory).
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t s_w[RB / 32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((int)lane >= o) x += y; }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < RB / 32 ? s_w[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if ((int)lane >= o) w += y; }
        if (lane < RB / 32) s_w[lane] = w;
    }
    __syncthreads();
    *total = s_w[RB / 32 - 1];
    return x - v + (warp ? s_w[warp - 1] : 0u);
}

// Single-CTA exclusive scan, in place, of the n block sums; *total_out = their sum.
__global__ void __launch_bounds__(1024) render_scan_sums_kernel(uint32_t n, uint32_t* __restrict__ sums, uint32_t* __restrict__ total_out) {
    __shared__ uint32_t s[1024];
    const uint32_t t = threadIdx.x, per = (n + 1023) / 1024;
    const uint32_t b = min(t * per, n), e = min(b + per, n);
    uint32_t sum = 0;
    for (uint32_t i = b; i < e; ++i) sum += sums[i];
    s[t] = sum;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {                                  // Hillis-Steele inclusive scan
        const uint32_t v = t >= off ? s[t - off] : 0u;
        __syncthreads();
        s[t] += v;
        __syncthreads();
    }
    uint32_t acc = s[t] - sum;
    for (uint32_t i = b; i < e; ++i) { const uint32_t v = sums[i]; sums[i] = acc; acc += v; }
    if (t == 1023) *total_out = s[1023];
}

// Order-preserving compaction: dst[scan] = src[k] (src == NULL: k) for every k < n with flags[k] != 0.
__global__ void __launch_bounds__(RB) render_compact_kernel(uint32_t n, const uint32_t* __restrict__ src, const uint32_t* __restrict__ flags,
                                                            const uint32_t* __restrict__ sums, uint32_t* __restrict__ dst) {
    const uint32_t k = blockIdx.x * RB + threadIdx.x;
    const uint32_t f = k < n ? flags[k] : 0u;
    uint32_t tot;
    const uint32_t pos = sums[blockIdx.x] + block_excl_scan(f, &tot);
    if (f) dst[pos] = src ? src[k] : k;
}

// Slab test, near distance and jitter of every ray (ray_sampler.h:29-48 through ray_setup).  Ray g draws its jitter where the tiled
// renderer would: tile g / tile, ray g % tile of that tile's ngp_march (each tile one rng.advance() further, ray_sampler.py:61).
__global__ void __launch_bounds__(RB) render_init_kernel(uint32_t n_rays, float lo, float hi, const float* __restrict__ rays_o,
                                                         const float* __restrict__ rays_d, float cone, float near_distance, MarchCfg c,
                                                         uint64_t rng_state, uint64_t rng_inc, uint32_t tile, float* __restrict__ ray_t,
                                                         uint32_t* __restrict__ ray_j, uint32_t* __restrict__ ray_step, float* __restrict__ ray_T,
                                                         float* __restrict__ rgb_out,
                                                         float* __restrict__ alpha_out, uint32_t* __restrict__ n_out,
                                                         uint32_t* __restrict__ flags, uint32_t* __restrict__ sums) {
    const uint32_t g = blockIdx.x * RB + threadIdx.x;
    uint32_t hit = 0;
    if (g < n_rays) {
        Pcg32 tile_rng{rng_state, rng_inc};
        tile_rng.advance((int64_t)((uint64_t)(g / tile) << 32));
        // ray_setup draws at (i + ray_offset) * 8: the wrapped offset makes that (g % tile) * 8
        const MarchRng mr{tile_rng.state, rng_inc, 0u - (g / tile) * tile};
        const RayState r = ray_setup(g, rays_o, rays_d, lo, hi, near_distance, cone, c, mr);
        hit = ray_tmin(lo, hi, r.o, r.d) != FLT_MAX ? 1u : 0u;
        ray_t[g] = r.startt;
        ray_j[g] = 0;
        ray_step[g] = 0;
        ray_T[g] = 1.f;
        rgb_out[3 * (size_t)g] = 0.f; rgb_out[3 * (size_t)g + 1] = 0.f; rgb_out[3 * (size_t)g + 2] = 0.f;
        alpha_out[g] = 0.f;
        n_out[g] = 0;
        flags[g] = hit;
    }
    uint32_t tot;
    block_excl_scan(hit, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

// March round: alive entry k < m continues the reference's loop (ray_sampler.h:50-72) from its saved t, sample count and step index for
// up to K samples, recording their t in its K slots of ts.  Every step of the t sequence, occupied or skipped, counts against
// MARCH_STEP_GUARD, as in march_count_kernel: a ray's samples are those with a step index below the guard, in both marches.
__global__ void __launch_bounds__(RB) render_march_kernel(uint32_t m, uint32_t K, const uint32_t* __restrict__ alive, float lo, float hi,
                                                          const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                          const uint8_t* __restrict__ bits, float cone, MarchCfg c, float* __restrict__ ray_t,
                                                          uint32_t* __restrict__ ray_j, uint32_t* __restrict__ ray_step, float* __restrict__ ts,
                                                          uint32_t* __restrict__ counts, uint32_t* __restrict__ sums) {
    const uint32_t k = blockIdx.x * RB + threadIdx.x;
    uint32_t n = 0;
    if (k < m) {
        const uint32_t g = alive[k];
        float o[3], d[3], id[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) { o[q] = rays_o[3 * (size_t)g + q]; d[q] = rays_d[3 * (size_t)g + q]; id[q] = 1.0f / d[q]; }
        float t = ray_t[g];
        uint32_t j = ray_j[g], step = ray_step[g];
        float* my_ts = ts + (size_t)k * K;
        while (n < K && step < MARCH_STEP_GUARD) {                                       // fewer than K samples: the march has ended
            const float p[3] = {__fmaf_rn(t, d[0], o[0]), __fmaf_rn(t, d[1], o[1]), __fmaf_rn(t, d[2], o[2])};
            if (!contains(lo, hi, p) || j >= NERF_STEPS) break;                         // while (aabb.contains(pos) && j < NERF_STEPS)
            const float dt = calc_dt(c, t, cone);
            const uint32_t mip = (uint32_t)mip_from_dt(c, dt, p[0], p[1], p[2]);
            if (occupied_at(p[0], p[1], p[2], bits, mip)) {
                my_ts[n++] = t;
                ++j;
                t += dt;
                ++step;
            } else {                                                                     // advance_to_next_voxel, step by step
                const float t_target = next_voxel_target(t, p, d, id, NERF_GRIDSIZE >> mip);
                do { t += calc_dt(c, t, cone); ++step; } while (t < t_target && step < MARCH_STEP_GUARD);
            }
        }
        ray_t[g] = t;
        ray_j[g] = j;
        ray_step[g] = step;
        counts[k] = n;
    }
    uint32_t tot;
    block_excl_scan(n, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

// The round's NerfCoordinate rows, dense in alive-list order (the row of march_emit_kernel: warped position, dt, direction).
__global__ void __launch_bounds__(RB) render_emit_kernel(uint32_t m, uint32_t K, const uint32_t* __restrict__ alive, float lo, float hi,
                                                         const float* __restrict__ rays_o, const float* __restrict__ rays_d, float cone,
                                                         MarchCfg c, const float* __restrict__ ts, const uint32_t* __restrict__ counts,
                                                         const uint32_t* __restrict__ sums, uint32_t* __restrict__ base_out,
                                                         float* __restrict__ rows) {
    const uint32_t k = blockIdx.x * RB + threadIdx.x;
    const uint32_t n = k < m ? counts[k] : 0u;
    uint32_t tot;
    const uint32_t base = sums[blockIdx.x] + block_excl_scan(n, &tot);
    if (k >= m) return;
    base_out[k] = base;
    if (n == 0) return;
    const uint32_t g = alive[k];
    float o[3], d[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) { o[q] = rays_o[3 * (size_t)g + q]; d[q] = rays_d[3 * (size_t)g + q]; }
    const float wd[3] = {(d[0] + 1.0f) * 0.5f, (d[1] + 1.0f) * 0.5f, (d[2] + 1.0f) * 0.5f}, diag = hi - lo;
    const float* my_ts = ts + (size_t)k * K;
    for (uint32_t s = 0; s < n; ++s) {
        const float t = my_ts[s];
        const float dt = calc_dt(c, t, cone);
        const float p[3] = {__fmaf_rn(t, d[0], o[0]), __fmaf_rn(t, d[1], o[1]), __fmaf_rn(t, d[2], o[2])};
        float* q = rows + (size_t)(base + s) * 7;
        q[0] = (p[0] - lo) / diag; q[1] = (p[1] - lo) / diag; q[2] = (p[2] - lo) / diag;   // warp_position
        q[3] = nerf_warp_dt(dt, c.cascades);
        q[4] = wd[0]; q[5] = wd[1]; q[6] = wd[2];
    }
}

// Composite round (calc_rgb.h:151-212 one sample after another, with the stopping rule).  Alive entries k >= m were not marched this
// round and stay alive unchanged.  flags[k] = 1: the ray goes on into the next round.
__global__ void __launch_bounds__(RB) render_composite_kernel(uint32_t n_alive, uint32_t m, uint32_t K, const uint32_t* __restrict__ alive,
                                                              const uint32_t* __restrict__ counts, const uint32_t* __restrict__ base_in,
                                                              const float* __restrict__ rows, const __half* __restrict__ net, uint32_t cascades,
                                                              float min_transmittance, float* __restrict__ ray_T, float* __restrict__ rgb_out,
                                                              float* __restrict__ alpha_out, uint32_t* __restrict__ n_out,
                                                              uint32_t* __restrict__ flags, uint32_t* __restrict__ sums) {
    const uint32_t k = blockIdx.x * RB + threadIdx.x;
    uint32_t go_on = 0;
    if (k < n_alive) {
        go_on = 1;
        if (k < m) {
            const uint32_t g = alive[k], n = counts[k], base = base_in[k];
            float T = ray_T[g];
            float rgb[3] = {rgb_out[3 * (size_t)g], rgb_out[3 * (size_t)g + 1], rgb_out[3 * (size_t)g + 2]};
            uint32_t done = n_out[g];
            bool stopped = false;
            for (uint32_t s = 0; s < n; ++s) {
                const uint2 u = __ldg(reinterpret_cast<const uint2*>(net) + base + s);
                const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
                const Sample smp = make_sample(make_float4(a.x, a.y, b.x, b.y), __ldg(rows + (size_t)(base + s) * 7 + 3), cascades);
                const float w = smp.alpha * T;
                rgb[0] = __fmaf_rn(w, smp.rgb[0], rgb[0]); rgb[1] = __fmaf_rn(w, smp.rgb[1], rgb[1]); rgb[2] = __fmaf_rn(w, smp.rgb[2], rgb[2]);
                T *= 1.f - smp.alpha;
                ++done;
                if (T < min_transmittance) { stopped = true; break; }                   // the rest of the ray cannot change the pixel
            }
            ray_T[g] = T;
            rgb_out[3 * (size_t)g] = rgb[0]; rgb_out[3 * (size_t)g + 1] = rgb[1]; rgb_out[3 * (size_t)g + 2] = rgb[2];
            alpha_out[g] = 1.f - T;
            n_out[g] = done;
            go_on = (!stopped && n == K) ? 1u : 0u;                                      // fewer than K samples: the march has ended
        }
        flags[k] = go_on;
    }
    uint32_t tot;
    block_excl_scan(go_on, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

struct RenderLayout {
    size_t ray_t, ray_j, ray_step, ray_T, alive, alive_next, counts, base, flags, sums, counters, ts, rows, net, bytes;
};
RenderLayout render_layout(uint32_t n_rays, uint32_t capacity) {
    RenderLayout L;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
    const size_t R = n_rays, C = capacity, nb = (R + RB - 1) / RB + 1;
    L.ray_t = take(4 * R); L.ray_j = take(4 * R); L.ray_step = take(4 * R); L.ray_T = take(4 * R);
    L.alive = take(4 * R); L.alive_next = take(4 * R);
    L.counts = take(4 * R); L.base = take(4 * R); L.flags = take(4 * R);
    L.sums = take(4 * nb); L.counters = take(16);
    L.ts = take(4 * C); L.rows = take(28 * C); L.net = take(8 * C);
    L.bytes = off;
    return L;
}
template <typename T> T* at(void* ws, size_t off) { return reinterpret_cast<T*>(static_cast<uint8_t*>(ws) + off); }

uint32_t blocks_for(uint32_t n) { return (n + RB - 1) / RB; }

// n_alive entries of the current list, their flags and block sums written: scan, compact into alive_next, read the count back, make
// alive_next the current list
int render_next_list(cudaStream_t s, void* ws, const RenderLayout& L, uint32_t n, const uint32_t* src, uint32_t* n_alive_host) {
    const uint32_t nb = blocks_for(n);
    uint32_t* counters = at<uint32_t>(ws, L.counters);
    render_scan_sums_kernel<<<1, 1024, 0, s>>>(nb, at<uint32_t>(ws, L.sums), counters + 1);
    NGP_LAUNCH_CHECK();
    render_compact_kernel<<<nb, RB, 0, s>>>(n, src, at<uint32_t>(ws, L.flags), at<uint32_t>(ws, L.sums), at<uint32_t>(ws, L.alive_next));
    NGP_LAUNCH_CHECK();
    NGP_CHECK_CUDA(cudaMemcpyAsync(n_alive_host, counters + 1, 4, cudaMemcpyDeviceToHost, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    if (*n_alive_host)
        NGP_CHECK_CUDA(cudaMemcpyAsync(at<uint32_t>(ws, L.alive), at<uint32_t>(ws, L.alive_next), (size_t)*n_alive_host * 4, cudaMemcpyDeviceToDevice, s));
    return 0;
}

}  // namespace

extern "C" {

int ngp_render_workspace_bytes(uint32_t n_rays, uint32_t capacity, uint64_t* layout_out) {
    NGP_REQUIRE(layout_out != nullptr, "ngp_render_workspace_bytes: layout_out is required");
    NGP_REQUIRE(capacity > 0, "ngp_render_workspace_bytes: the row capacity must be positive");
    const RenderLayout L = render_layout(n_rays, capacity);
    layout_out[0] = L.bytes;
    layout_out[1] = L.rows;
    layout_out[2] = L.net;
    layout_out[3] = L.counters;
    return 0;
}

int ngp_render_init(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, float aabb_lo, float aabb_hi, const float* rays_o,
                    const float* rays_d, float cone_angle, float near_distance, uint32_t cascades, int const_dt, uint64_t rng_state,
                    uint64_t rng_inc, uint32_t jitter_tile, float* rgb_out, float* alpha_out, uint32_t* n_samples_out, uint32_t* n_alive_host) {
    NGP_REQUIRE(capacity > 0, "ngp_render_init: the row capacity must be positive");
    NGP_REQUIRE(workspace != nullptr, "ngp_render_init: workspace is required (ngp_render_workspace_bytes)");
    NGP_REQUIRE(jitter_tile > 0, "ngp_render_init: jitter_tile must be positive");
    NGP_REQUIRE(cascades >= 1 && cascades <= 8, "ngp_render_init: cascades out of range");
    NGP_REQUIRE(n_alive_host != nullptr, "ngp_render_init: n_alive_host is required");
    *n_alive_host = 0;
    if (n_rays == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const RenderLayout L = render_layout(n_rays, capacity);
    const MarchCfg c = make_cfg(cascades, const_dt);
    render_init_kernel<<<blocks_for(n_rays), RB, 0, s>>>(n_rays, aabb_lo, aabb_hi, rays_o, rays_d, cone_angle, near_distance, c, rng_state, rng_inc,
                                                         jitter_tile, at<float>(workspace, L.ray_t), at<uint32_t>(workspace, L.ray_j), at<uint32_t>(workspace, L.ray_step),
                                                         at<float>(workspace, L.ray_T), rgb_out, alpha_out, n_samples_out,
                                                         at<uint32_t>(workspace, L.flags), at<uint32_t>(workspace, L.sums));
    NGP_LAUNCH_CHECK();
    return render_next_list(s, workspace, L, n_rays, nullptr, n_alive_host);
}

int ngp_render_march_round(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps, float aabb_lo,
                           float aabb_hi, const float* rays_o, const float* rays_d, const uint8_t* bitfield, float cone_angle, uint32_t cascades,
                           int const_dt) {
    NGP_REQUIRE(capacity > 0, "ngp_render_march_round: the row capacity must be positive");
    NGP_REQUIRE(workspace != nullptr, "ngp_render_march_round: workspace is required (ngp_render_workspace_bytes)");
    NGP_REQUIRE(k_steps >= 1 && k_steps <= capacity, "ngp_render_march_round: k_steps must be in [1, capacity]");
    NGP_REQUIRE(n_alive <= n_rays, "ngp_render_march_round: n_alive exceeds n_rays");
    NGP_REQUIRE(cascades >= 1 && cascades <= 8, "ngp_render_march_round: cascades out of range");
    cudaStream_t s = (cudaStream_t)stream;
    const RenderLayout L = render_layout(n_rays, capacity);
    uint32_t* counters = at<uint32_t>(workspace, L.counters);
    NGP_CHECK_CUDA(cudaMemsetAsync(counters, 0, 4, s));
    if (n_alive == 0) return 0;
    const uint32_t m = min(n_alive, capacity / k_steps);                                  // m * K rows fit the capacity
    const MarchCfg c = make_cfg(cascades, const_dt);
    const uint32_t nb = blocks_for(m);
    render_march_kernel<<<nb, RB, 0, s>>>(m, k_steps, at<uint32_t>(workspace, L.alive), aabb_lo, aabb_hi, rays_o, rays_d, bitfield, cone_angle, c,
                                          at<float>(workspace, L.ray_t), at<uint32_t>(workspace, L.ray_j), at<uint32_t>(workspace, L.ray_step), at<float>(workspace, L.ts),
                                          at<uint32_t>(workspace, L.counts), at<uint32_t>(workspace, L.sums));
    NGP_LAUNCH_CHECK();
    render_scan_sums_kernel<<<1, 1024, 0, s>>>(nb, at<uint32_t>(workspace, L.sums), counters);
    NGP_LAUNCH_CHECK();
    render_emit_kernel<<<nb, RB, 0, s>>>(m, k_steps, at<uint32_t>(workspace, L.alive), aabb_lo, aabb_hi, rays_o, rays_d, cone_angle, c,
                                         at<float>(workspace, L.ts), at<uint32_t>(workspace, L.counts), at<uint32_t>(workspace, L.sums),
                                         at<uint32_t>(workspace, L.base), at<float>(workspace, L.rows));
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_render_composite_round(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps,
                               float min_transmittance, uint32_t cascades, float* rgb_out, float* alpha_out, uint32_t* n_samples_out,
                               uint32_t* n_alive_host) {
    NGP_REQUIRE(capacity > 0, "ngp_render_composite_round: the row capacity must be positive");
    NGP_REQUIRE(workspace != nullptr, "ngp_render_composite_round: workspace is required (ngp_render_workspace_bytes)");
    NGP_REQUIRE(k_steps >= 1 && k_steps <= capacity, "ngp_render_composite_round: k_steps must be in [1, capacity]");
    NGP_REQUIRE(n_alive <= n_rays, "ngp_render_composite_round: n_alive exceeds n_rays");
    NGP_REQUIRE(n_alive_host != nullptr, "ngp_render_composite_round: n_alive_host is required");
    *n_alive_host = 0;
    if (n_alive == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const RenderLayout L = render_layout(n_rays, capacity);
    const uint32_t m = min(n_alive, capacity / k_steps);
    render_composite_kernel<<<blocks_for(n_alive), RB, 0, s>>>(n_alive, m, k_steps, at<uint32_t>(workspace, L.alive), at<uint32_t>(workspace, L.counts),
                                                               at<uint32_t>(workspace, L.base), at<float>(workspace, L.rows),
                                                               at<__half>(workspace, L.net), cascades, min_transmittance, at<float>(workspace, L.ray_T),
                                                               rgb_out, alpha_out, n_samples_out, at<uint32_t>(workspace, L.flags),
                                                               at<uint32_t>(workspace, L.sums));
    NGP_LAUNCH_CHECK();
    return render_next_list(s, workspace, L, n_alive, at<uint32_t>(workspace, L.alive), n_alive_host);
}

}  // extern "C"
