// R5/R6/R8/R9: occupancy-grid ray march, compaction and volume-render composite (forward / backward /
// inference / fused training tail).  Compiled with -fmad=false: every multiply-add that the reference's GPU build
// contracts is written as an explicit __fmaf_rn so the sample sequence is reproducible op-for-op by the oracle
// (oracle/ngp_oracle.c, fma_mode 1) and sample indices stay bit-exact (SURVEY.md H4).
//
// March (replaces DGS/op_header/ray_sampler.h:4-114): pass 1 counts steps per ray, a single-CTA scan turns the
// counts into ray-ordered bases (deterministic; the reference claims ranges with atomicAdd), pass 2 emits the
// NerfCoordinate rows.  No 117 MB memset (DGS/ray_sampler.py:50), no host sync (:65,70).
#include "march_common.cuh"
#include <cfloat>
#include <cstdlib>

int* ngp_err_flag();

namespace {

// One marching pass by a whole warp per ray; EMIT=false counts, EMIT=true writes rows.
//
// The reference's loop visits a fixed sequence t_{k+1} = t_k + calc_dt(t_k) that does not depend on the occupancy
// (both its branches advance by calc_dt; the empty-space branch just advances several steps without testing).  The warp
// therefore materialises 32 consecutive t_k (same float additions, same order), evaluates position, mip level, occupancy
// bit and the distance to the next voxel of all 32 in parallel, and then replays the reference's sequential control flow
// on two ballot masks -- identical arithmetic per visited step, 32 occupancy lookups in flight instead of one.
//
// This monolithic form (everything of a ray in one warp's serial loop) is the FALLBACK for rays with more than MARCH_MAXC chunks;
// the production path below splits the same computation into a chunk evaluation pass and a replay pass.
template <bool EMIT>
__device__ __forceinline__ uint32_t march_ray_warp(const RayState& r, float lo, float hi, float cone, const MarchCfg& c,
                                                   const uint8_t* __restrict__ bits, uint32_t limit, float* __restrict__ out) {
    const uint32_t lane = threadIdx.x & 31;
    const unsigned FULL = 0xffffffffu;
    uint32_t j = 0;
    float t0 = r.startt;          // t of lane 0 of the current chunk
    bool pending = false;         // an empty-space skip that did not finish inside the previous chunk
    float pending_tt = 0.f;
    float wd[3], diag = hi - lo;
    if (EMIT) { wd[0] = (r.d[0] + 1.0f) * 0.5f; wd[1] = (r.d[1] + 1.0f) * 0.5f; wd[2] = (r.d[2] + 1.0f) * 0.5f; }
    uint32_t chunk = 0;
    for (uint32_t guard = 0; guard < (1u << 20); ++guard) {   // a degenerate ray (d == 0) would spin forever in the reference
        float t = t0;
        for (uint32_t i = 0; i < lane; ++i) t += calc_dt(c, t, cone);          // t_k .. t_{k+31}, sequential float adds
        const float dt = calc_dt(c, t, cone);
        const float t_next_chunk = __shfl_sync(FULL, t + dt, 31);
        int cur = 0;
        if (pending) {
            const uint32_t ge = __ballot_sync(FULL, !(t < pending_tt));
            if (ge == 0) {                                                      // the whole chunk lies inside the skipped span
                ++chunk;
                t0 = t_next_chunk;
                continue;
            }
            cur = __ffs(ge) - 1;
            pending = false;
        }
        const float p[3] = {__fmaf_rn(t, r.d[0], r.o[0]), __fmaf_rn(t, r.d[1], r.o[1]), __fmaf_rn(t, r.d[2], r.o[2])};
        const bool inside = contains(lo, hi, p);
        uint32_t mip = 0;
        bool occ = false;
        float t_target = 0.f;
        if (inside) {
            mip = (uint32_t)mip_from_dt(c, dt, p[0], p[1], p[2]);
            occ = occupied_at(p[0], p[1], p[2], bits, mip);
            if (!occ) {                                                          // distance_to_next_voxel, ray_sampler_header.h:728-739
                const float rs = (float)(NERF_GRIDSIZE >> mip);
                const float q[3] = {rs * p[0], rs * p[1], rs * p[2]};
                const float tx = (floorf(q[0] + 0.5f + 0.5f * sgn(r.d[0])) - q[0]) * r.id[0];
                const float ty = (floorf(q[1] + 0.5f + 0.5f * sgn(r.d[1])) - q[1]) * r.id[1];
                const float tz = (floorf(q[2] + 0.5f + 0.5f * sgn(r.d[2])) - q[2]) * r.id[2];
                t_target = t + fmaxf(fminf(fminf(tx, ty), tz) / rs, 0.0f);
            }
        }
        const uint32_t inside_m = __ballot_sync(FULL, inside), occ_m = __ballot_sync(FULL, occ);
        bool done = false;
        uint32_t emit_m = 0;
        while (cur < 32) {
            if (!((inside_m >> cur) & 1u) || j >= limit) { done = true; break; }   // while (aabb.contains(pos) && j < limit)
            if ((occ_m >> cur) & 1u) {
                const uint32_t run_m = (occ_m & inside_m) >> cur;                 // consecutive occupied steps are taken one by one
                uint32_t n_run = (run_m == 0xffffffffu) ? 32u : (uint32_t)__ffs(~run_m) - 1u;
                n_run = min(n_run, limit - j);
                emit_m |= (n_run >= 32u ? 0xffffffffu : ((1u << n_run) - 1u)) << cur;
                if (EMIT && (int)lane >= cur && lane < cur + n_run) {
                    float* q = out + (size_t)(j + lane - cur) * 7;
                    q[0] = (p[0] - lo) / diag; q[1] = (p[1] - lo) / diag; q[2] = (p[2] - lo) / diag;   // warp_position
                    q[3] = nerf_warp_dt(dt, c.cascades);
                    q[4] = wd[0]; q[5] = wd[1]; q[6] = wd[2];
                }
                j += n_run;
                cur += n_run;
            } else {
                // advance_to_next_voxel: do { t += dt } while (t < t_target)  -> first later step with !(t < t_target)
                const float tt = __shfl_sync(FULL, t_target, cur);
                uint32_t ge = __ballot_sync(FULL, !(t < tt));
                ge &= (cur >= 31) ? 0u : ~((2u << cur) - 1u);
                if (ge) cur = __ffs(ge) - 1;
                else { pending = true; pending_tt = tt; cur = 32; }
            }
        }
        ++chunk;
        if (done) break;
        t0 = t_next_chunk;
    }
    return j;
}

// ---- producer / consumer march --------------------------------------------------------------------------------------------------
// Round 1 ran the whole loop above per ray in one warp: ~1.2 k cycles per 32-step chunk, 40-64 chunks in sequence, and the kernel
// lasted as long as its longest ray (80 us for ~2 200 rays at 16 % of the warp slots).  Everything in a chunk except the replay of the
// control flow is independent of every other chunk -- the t sequence is fixed, and position / mip level / occupancy bit / distance to
// the next voxel are functions of t alone.  march_count_kernel therefore runs TWO warps per ray:
//   producer: walks the t sequence (the same float additions in the same order; lane k keeps t_k of the current chunk), evaluates the
//             32 steps of every chunk and pushes {inside mask, occupied mask, per step t, skip target t_target, in-chunk skip
//             destination} into a 4-slot ring in shared memory.  No control flow depends on loaded data: the occupancy byte of a
//             chunk is tested while the next chunk's lookup is in flight (two chunk states in ping-pong registers);
//   consumer: the reference's sequential control flow (ray_sampler.h:50-72) replayed on the masks -- a few integer operations and one
//             shuffle per visited run / skip -- and, for every chunk that emits samples, {t values, emit mask, first ray-local
//             index} appended to the ray's emit list in global memory.
// Hand-over through mbarriers (FULL / EMPTY per slot).  After the scan, march_emit_kernel (CTA per ray, warp per list entry) turns
// the list into rows.  Same arithmetic per visited step as the reference, hence the same samples bit for bit
// (tests/test_gpu_ops.py::test_march_bit_exact).
constexpr uint32_t MARCH_SLOTS = 4;
constexpr uint32_t MARCH_EMIT_CAP = 64;        // emitting chunks recorded per ray (a 1024-sample ray of solid runs needs 33); more -> re-march
constexpr uint32_t MARCH_CHUNK_GUARD = MARCH_STEP_GUARD / 32;   // a degenerate ray (d == 0, NaN) would never leave the box: forced terminal chunk
struct __align__(16) EmitRec { float t[32]; uint32_t mask, j0, pad0, pad1; };
static_assert(sizeof(EmitRec) == 144, "EmitRec must be 144 bytes");
constexpr size_t MARCH_RAY_BYTES = (size_t)MARCH_EMIT_CAP * sizeof(EmitRec);

struct __align__(16) RingSlot {
    uint32_t inside, occ, terminal;
    float t0_next;                 // t of the first step of the NEXT chunk (every t of this chunk is smaller)
    uint8_t dest[32];              // first lane > l with !(t < t_target[l]) inside the chunk, 32 = beyond the chunk
    float t[32];
    float tt[32];                  // t_target of empty steps (distance_to_next_voxel)
};
struct RayRing {
    uint64_t full[MARCH_SLOTS], empty[MARCH_SLOTS];
    RingSlot slot[MARCH_SLOTS];
};

__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr_u32(bar)) : "memory");
}
// bounded wait (a protocol mistake must not hang the GPU box): false on timeout
__device__ __forceinline__ bool mb_wait(uint64_t* bar, uint32_t parity) {
#pragma unroll 1
    for (uint32_t spin = 0; spin < (1u << 24); ++spin) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_addr_u32(bar)), "r"(parity) : "memory");
        if (ok) return true;
    }
    return false;
}

struct ChunkState {           // per lane: one step of a chunk between the two halves of the evaluation
    float t0_next, t, dt, p[3];
    uint32_t inside_m, mip, byte, bit;
    bool inside;
};

constexpr int MARCH_RAYS_PER_CTA = 4;
__global__ void __launch_bounds__(64 * MARCH_RAYS_PER_CTA)
march_count_kernel(uint32_t n_rays, float lo, float hi, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                   const uint8_t* __restrict__ bits, float cone, float near_distance, MarchCfg c, MarchRng mr,
                   uint8_t* __restrict__ ws, uint32_t* __restrict__ counts, uint32_t* __restrict__ n_emit, int* __restrict__ err) {
    __shared__ RayRing s_ring[MARCH_RAYS_PER_CTA];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rl = warp % MARCH_RAYS_PER_CTA;                    // ray slot of this warp inside the CTA
    const bool producer = warp < MARCH_RAYS_PER_CTA;
    const uint32_t i = blockIdx.x * MARCH_RAYS_PER_CTA + rl;
    RayRing& ring = s_ring[rl];
    if (producer && lane == 0) {
        for (uint32_t k = 0; k < MARCH_SLOTS; ++k) { mb_init(&ring.full[k], 1); mb_init(&ring.empty[k], 1); }
    }
    __syncthreads();
    if (i >= n_rays) return;
    const unsigned FULL = 0xffffffffu;

    if (producer) {
        const RayState r = ray_setup(i, rays_o, rays_d, lo, hi, near_distance, cone, c, mr);
        float tc = r.startt;                 // running t of the sequence (identical in all lanes)
        // first half of a chunk: t values, positions, occupancy lookup issued (not consumed)
        auto stage1 = [&](ChunkState& st) {
            float t = tc;
            bool closed = false;
            if (c.const_dt) {
                // t_{k+1} = fl(t_k + h) with a constant h: while the sequence stays inside one binade every t_k is a multiple of the
                // binade's ulp, so every addition rounds h to the same multiple q of that ulp (unless h lies exactly half way between
                // two multiples, where round-to-even looks at t_k) and t_k = t_0 + k q exactly.  Then lane k gets t_k from ONE fma
                // (k q < 2^24 ulp: exact) instead of k dependent additions.  Any chunk that crosses a power of two, or a tie, takes the
                // sequential path below.
                const float h = c.min_cone * 0.5f;
                const float q = (tc + h) - tc;                                    // exact (Sterbenz)
                const float t_end = __fmaf_rn(32.0f, q, tc);
                const uint32_t e0 = __float_as_uint(tc) >> 23, e1 = __float_as_uint(t_end) >> 23;
                const float r = h * __uint_as_float((277u - e0) << 23);          // h / ulp(tc) = h * 2^(150 - e0), exact scaling
                if (e0 == e1 && e0 >= 117u && e0 <= 140u && (r - floorf(r)) != 0.5f) {
                    t = __fmaf_rn((float)lane, q, tc);
                    tc = t_end;
                    closed = true;
                }
            }
            if (!closed) {
#pragma unroll
                for (int k = 0; k < 32; ++k) {                                    // t_k .. t_{k+31}: the reference's float additions, in order
                    if ((int)lane == k) t = tc;
                    tc += calc_dt(c, tc, cone);
                }
            }
            st.t0_next = tc;
            st.t = t;
            st.dt = calc_dt(c, t, cone);
            st.p[0] = __fmaf_rn(t, r.d[0], r.o[0]); st.p[1] = __fmaf_rn(t, r.d[1], r.o[1]); st.p[2] = __fmaf_rn(t, r.d[2], r.o[2]);
            st.inside = contains(lo, hi, st.p);
            st.inside_m = __ballot_sync(FULL, st.inside);
            st.mip = 0; st.byte = 0; st.bit = 0;
            if (st.inside) {                                                       // occupied_at(): load now, test in the second half
                st.mip = (uint32_t)mip_from_dt(c, st.dt, st.p[0], st.p[1], st.p[2]);
                const uint32_t idx = grid_idx_at(st.p[0], st.p[1], st.p[2], st.mip);
                st.byte = __ldg(bits + idx / 8 + (NERF_GRID_N / 8) * st.mip);
                st.bit = 1u << (idx % 8);
            }
        };
        // second half: occupancy test, skip target, in-chunk skip destination; push into the ring.  false = hand-over timed out
        auto stage2 = [&](const ChunkState& st, uint32_t ch, bool terminal) -> bool {
            const bool occ = st.inside && (st.byte & st.bit) != 0;
            const uint32_t occ_m = __ballot_sync(FULL, occ);
            float tt = 0.f;
            if (st.inside && !occ) {                                               // distance_to_next_voxel, ray_sampler_header.h:728-739
                const float rs = (float)(NERF_GRIDSIZE >> st.mip);
                const float q[3] = {rs * st.p[0], rs * st.p[1], rs * st.p[2]};
                const float tx = (floorf(q[0] + 0.5f + 0.5f * sgn(r.d[0])) - q[0]) * r.id[0];
                const float ty = (floorf(q[1] + 0.5f + 0.5f * sgn(r.d[1])) - q[1]) * r.id[1];
                const float tz = (floorf(q[2] + 0.5f + 0.5f * sgn(r.d[2])) - q[2]) * r.id[2];
                const float rs_inv = __uint_as_float((120u + st.mip) << 23);      // 1 / rs = 2^(mip - 7): x / rs == x * rs_inv bit for bit
                tt = st.t + fmaxf(fminf(fminf(tx, ty), tz) * rs_inv, 0.0f);
            }
            // advance_to_next_voxel: do { t += dt } while (t < t_target) = the first later step with !(t < t_target); t increases
            // with the lane, so that step is found by bisection over the lanes (5 shuffles instead of a ballot per source lane)
            uint32_t lo_l = lane + 1, hi_l = 32;
#pragma unroll
            for (int it = 0; it < 5; ++it) {
                const uint32_t mid = (lo_l + hi_l) >> 1;
                const float tm = __shfl_sync(FULL, st.t, mid & 31);
                const bool less = mid < 32 && tm < tt;
                if (lo_l < hi_l) { if (less) lo_l = mid + 1; else hi_l = mid; }
            }
            const uint32_t k = ch % MARCH_SLOTS;
            if (!mb_wait(&ring.empty[k], ((ch / MARCH_SLOTS) & 1u) ^ 1u)) return false;   // the consumer has released this slot
            RingSlot& sl = ring.slot[k];
            if (lane == 0) { sl.inside = st.inside_m; sl.occ = occ_m; sl.terminal = terminal ? 1u : 0u; sl.t0_next = st.t0_next; }
            sl.dest[lane] = (uint8_t)lo_l;
            sl.t[lane] = st.t;
            sl.tt[lane] = tt;
            __syncwarp();
            if (lane == 0) mb_arrive(&ring.full[k]);
            return true;
        };
        // two chunk states in ping-pong: no register copy ever waits for a lookup that is still in flight
        ChunkState A, B;
        uint32_t ch = 0;
        bool ok = true;
        stage1(A);
        bool a_term = A.inside_m == 0, b_term = false;
        for (;;) {
            const bool b_valid = !a_term;
            if (b_valid) { stage1(B); b_term = B.inside_m == 0 || ch + 2 >= MARCH_CHUNK_GUARD; }
            ok = stage2(A, ch++, a_term);
            if (!ok || !b_valid) break;
            const bool a_valid = !b_term;
            if (a_valid) { stage1(A); a_term = A.inside_m == 0 || ch + 2 >= MARCH_CHUNK_GUARD; }
            ok = stage2(B, ch++, b_term);
            if (!ok || !a_valid) break;
        }
        if (!ok && lane == 0) atomicExch(err, 3);
    } else {
        // ---- consumer: ray_sampler.h:50-72 on the masks
        EmitRec* elist = reinterpret_cast<EmitRec*>(ws + (size_t)i * MARCH_RAY_BYTES);
        const uint32_t limit = NERF_STEPS;
        uint32_t j = 0, ne = 0;
        bool pending = false, finished = false, ok = true;
        float pending_tt = 0.f;
        for (uint32_t ch = 0;; ++ch) {
            const uint32_t k = ch % MARCH_SLOTS;
            if (!mb_wait(&ring.full[k], (ch / MARCH_SLOTS) & 1u)) { ok = false; break; }
            const RingSlot& sl = ring.slot[k];
            const uint32_t inside_m = sl.inside, occ_m = sl.occ, terminal = sl.terminal;
            if (!finished) {
                int cur = 0;
                uint32_t emit_m = 0;
                const uint32_t j0 = j;
                bool skip = false;
                if (pending) {
                    if (!(pending_tt < sl.t0_next) && !terminal) skip = true;       // every t of this chunk < t0 of the next <= target
                    else {
                        const uint32_t ge = __ballot_sync(FULL, !(sl.t[lane] < pending_tt));
                        if (ge == 0) skip = true;
                        else { cur = __ffs(ge) - 1; pending = false; }
                    }
                }
                if (!skip) {
                    const uint32_t d = sl.dest[lane];
                    while (cur < 32) {
                        if (!((inside_m >> cur) & 1u) || j >= limit) { finished = true; break; }   // while (aabb.contains(pos) && j < NERF_STEPS)
                        if ((occ_m >> cur) & 1u) {
                            const uint32_t run_m = (occ_m & inside_m) >> cur;             // consecutive occupied steps are taken one by one
                            uint32_t n_run = (run_m == 0xffffffffu) ? 32u : (uint32_t)__ffs(~run_m) - 1u;
                            n_run = min(n_run, limit - j);
                            emit_m |= (n_run >= 32u ? 0xffffffffu : ((1u << n_run) - 1u)) << cur;
                            j += n_run;
                            cur += n_run;
                        } else {
                            const uint32_t dc = __shfl_sync(FULL, d, cur);
                            if (dc < 32) cur = (int)dc;
                            else { pending = true; pending_tt = sl.tt[cur]; cur = 32; }
                        }
                    }
                }
                if (emit_m) {                                                      // this chunk emits: append to the ray's emit list
                    if (ne < MARCH_EMIT_CAP) {
                        elist[ne].t[lane] = sl.t[lane];
                        if (lane == 0) { elist[ne].mask = emit_m; elist[ne].j0 = j0; }
                    }
                    ++ne;
                }
            }
            __syncwarp();
            if (lane == 0) mb_arrive(&ring.empty[k]);                              // (after `finished` the remaining chunks are only drained)
            if (terminal) break;
        }
        if (!ok && lane == 0) atomicExch(err, 3);
        if (lane == 0) { counts[i] = j; n_emit[i] = ne; }
    }
}

// Single-CTA exclusive scan over ray counts (R <= a few 100k): numsteps[i] = {count or 0, base}, ray index of accepted rays.
__global__ void __launch_bounds__(1024) march_scan_kernel(uint32_t n_rays, uint32_t max_samples, const uint32_t* __restrict__ counts,
                                                          uint32_t* __restrict__ numsteps, uint32_t* __restrict__ ray_indices,
                                                          uint32_t* __restrict__ counters) {
    __shared__ uint32_t s_sum[1024], s_acc[1024];
    const uint32_t t = threadIdx.x;
    const uint32_t per = (n_rays + 1023) / 1024;
    const uint32_t b = t * per, e = min(b + per, n_rays);
    uint32_t sum = 0;
    for (uint32_t i = b; i < e; ++i) sum += counts[i];
    s_sum[t] = sum;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {           // Hillis-Steele inclusive scan
        uint32_t v = (t >= off) ? s_sum[t - off] : 0;
        __syncthreads();
        s_sum[t] += v;
        __syncthreads();
    }
    uint32_t base = s_sum[t] - sum, acc = 0;
    for (uint32_t i = b; i < e; ++i) {
        const uint32_t n = counts[i];
        const bool ok = base + n <= max_samples;                 // ray_sampler.h:74-80
        numsteps[2 * i] = ok ? n : 0;
        numsteps[2 * i + 1] = base;
        acc += ok ? 1 : 0;
        base += n;
    }
    s_acc[t] = acc;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {
        uint32_t v = (t >= off) ? s_acc[t - off] : 0;
        __syncthreads();
        s_acc[t] += v;
        __syncthreads();
    }
    uint32_t ridx = s_acc[t] - acc;
    base = s_sum[t] - sum;
    for (uint32_t i = b; i < e; ++i) {
        const uint32_t n = counts[i];
        const bool ok = base + n <= max_samples;
        if (ok) ray_indices[i] = (n == 0) ? 0xFFFFFFFFu : ridx;  // :84-93
        ridx += ok ? 1 : 0;
        base += n;
    }
    if (t == 1023) { counters[0] = s_acc[1023]; counters[1] = s_sum[1023]; }
}

// Emit pass: one CTA per ray, one warp per entry of the ray's emit list.  The rows of a chunk are contiguous in the output
// (ray-ordered, the replay left the ray-local index of the chunk's first sample), so they are staged in shared memory and written as
// one coalesced block of n x 7 floats instead of 7 strided 4-byte stores per lane.  A ray whose list overflowed is re-marched.
__global__ void __launch_bounds__(128) march_emit_kernel(uint32_t n_rays, float lo, float hi, const float* __restrict__ rays_o,
                                                         const float* __restrict__ rays_d, const uint8_t* __restrict__ bits, float cone,
                                                         float near_distance, MarchCfg c, MarchRng mr,
                                                         const uint32_t* __restrict__ numsteps, float* __restrict__ coords,
                                                         const uint8_t* __restrict__ ws, const uint32_t* __restrict__ n_emit) {
    __shared__ float s_rows[4][32 * 7];
    const uint32_t i = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n = numsteps[2 * i], base = numsteps[2 * i + 1];
    if (n == 0) return;
    float* out = coords + (size_t)base * 7;
    const uint32_t ne = n_emit[i];
    if (ne > MARCH_EMIT_CAP) {
        if (warp == 0) {
            const RayState r = ray_setup(i, rays_o, rays_d, lo, hi, near_distance, cone, c, mr);
            march_ray_warp<true>(r, lo, hi, cone, c, bits, n, out);
        }
        return;
    }
    const EmitRec* elist = reinterpret_cast<const EmitRec*>(ws + (size_t)i * MARCH_RAY_BYTES);
    float o[3], d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { o[k] = rays_o[3 * (size_t)i + k]; d[k] = rays_d[3 * (size_t)i + k]; }
    const float wd[3] = {(d[0] + 1.0f) * 0.5f, (d[1] + 1.0f) * 0.5f, (d[2] + 1.0f) * 0.5f}, diag = hi - lo;
    float* rows = s_rows[warp];
    for (uint32_t e = warp; e < ne; e += 4) {
        const uint32_t mask = elist[e].mask, j0 = elist[e].j0, cnt = __popc(mask);
        if ((mask >> lane) & 1u) {
            const float t = elist[e].t[lane];
            const float dt = calc_dt(c, t, cone);
            const float p[3] = {__fmaf_rn(t, d[0], o[0]), __fmaf_rn(t, d[1], o[1]), __fmaf_rn(t, d[2], o[2])};
            float* q = rows + __popc(mask & ((1u << lane) - 1u)) * 7;
            q[0] = (p[0] - lo) / diag; q[1] = (p[1] - lo) / diag; q[2] = (p[2] - lo) / diag;   // warp_position
            q[3] = nerf_warp_dt(dt, c.cascades);
            q[4] = wd[0]; q[5] = wd[1]; q[6] = wd[2];
        }
        __syncwarp();
        float* dst = out + (size_t)j0 * 7;
        for (uint32_t k = lane; k < cnt * 7; k += 32) dst[k] = rows[k];
        __syncwarp();
    }
}

// Compaction bases: exclusive scan of the per-ray counts in ray order (single CTA), with the reference's truncation rule.
__global__ void __launch_bounds__(1024) compact_scan_kernel(uint32_t n_rays, uint32_t max_compacted, const uint32_t* __restrict__ numsteps_in,
                                                            uint32_t* __restrict__ numsteps_out, uint32_t* __restrict__ counters) {
    __shared__ uint32_t s_sum[1024], s_acc[1024];
    const uint32_t t = threadIdx.x;
    const uint32_t per = (n_rays + 1023) / 1024;
    const uint32_t b = min(t * per, n_rays), e = min(b + per, n_rays);
    uint32_t sum = 0;
    for (uint32_t i = b; i < e; ++i) sum += numsteps_in[2 * i];
    s_sum[t] = sum;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {
        uint32_t v = (t >= off) ? s_sum[t - off] : 0;
        __syncthreads();
        s_sum[t] += v;
        __syncthreads();
    }
    uint32_t base = s_sum[t] - sum, acc = 0;
    for (uint32_t i = b; i < e; ++i) {
        const uint32_t n = numsteps_in[2 * i];
        const uint32_t cn = min(max_compacted - min(max_compacted, base), n);      // compacted_coord.h:62-63
        numsteps_out[2 * i] = cn;
        numsteps_out[2 * i + 1] = base;
        acc += cn ? 1 : 0;
        base += n;
    }
    s_acc[t] = acc;
    __syncthreads();
    if (t == 0) {
        uint32_t rays = 0;
        for (int k = 0; k < 1024; ++k) rays += s_acc[k];
        counters[0] = s_sum[1023];
        counters[1] = rays;
    }
}
// one warp per ray copies its rows from the raw base to the compacted base
__global__ void compact_copy_kernel(uint32_t n_rays, const float* __restrict__ coords_in, const uint32_t* __restrict__ numsteps_in,
                                    float* __restrict__ coords_out, const uint32_t* __restrict__ numsteps_out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n_rays) return;
    const uint32_t base = numsteps_in[2 * warp + 1], cn = numsteps_out[2 * warp], cbase = numsteps_out[2 * warp + 1];
    for (uint32_t k = lane; k < cn * 7; k += 32) coords_out[(size_t)cbase * 7 + k] = coords_in[(size_t)base * 7 + k];
}
__global__ void zero_tail_kernel(float* __restrict__ coords_out, const uint32_t* __restrict__ counters, uint32_t max_compacted) {
    const uint32_t total = min(counters[0], max_compacted);
    const size_t b = (size_t)total * 7, e = (size_t)max_compacted * 7;
    for (size_t k = b + blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < e; k += (size_t)gridDim.x * blockDim.x) coords_out[k] = 0.f;
}

// ---- composite -------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ void store_net(T* dst, size_t k, float4 v);
template <> __device__ __forceinline__ void store_net<float>(float* dst, size_t k, float4 v) { reinterpret_cast<float4*>(dst)[k] = v; }
template <> __device__ __forceinline__ void store_net<__half>(__half* dst, size_t k, float4 v) {
    __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(dst)[k] = u;
}

// Lane l handles samples l, l+32, ... of its ray.  Transmittance T_j = prod_{k<j}(1-alpha_k) and the running colour are
// warp scans (the reference accumulates them serially per thread, calc_rgb.h:45-65): same formulae, reassociated sums.
__device__ __forceinline__ float warp_incl_prod(float v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if ((int)lane >= o) v *= u; }
    return v;
}
__device__ __forceinline__ float warp_incl_sum(float v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if ((int)lane >= o) v += u; }
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// A ray is one warp's loop over its samples, and the kernel lasts as long as its longest ray (all rays of a batch are resident at
// once; ncu: 7 % of the warp slots active on average), i.e. as long as that ray's chain of warp scans.  Each lane therefore owns
// COMP_K CONSECUTIVE samples of a 32 x COMP_K chunk: the products / sums over its own samples are plain register arithmetic, and
// one warp scan over the lane totals serves COMP_K x 32 samples -- a 1024-sample ray is 8 scan rounds instead of 32.  The loads of
// the next chunk are issued before the current one is evaluated (raw rows in a register set of their own).
constexpr int COMP_K = 4;
template <typename T> struct NetRow;
template <> struct NetRow<float> { float4 v; };
template <> struct NetRow<__half> { uint2 v; };
__device__ __forceinline__ void load_row(const float* net, size_t k, NetRow<float>* r) { r->v = __ldg(reinterpret_cast<const float4*>(net) + k); }
__device__ __forceinline__ void load_row(const __half* net, size_t k, NetRow<__half>* r) { r->v = __ldg(reinterpret_cast<const uint2*>(net) + k); }
__device__ __forceinline__ void zero_row(NetRow<float>* r) { r->v = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void zero_row(NetRow<__half>* r) { r->v = make_uint2(0u, 0u); }
__device__ __forceinline__ float4 row_f4(const NetRow<float>& r) { return r.v; }
__device__ __forceinline__ float4 row_f4(const NetRow<__half>& r) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&r.v.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
template <typename T> struct ChunkRaw {
    NetRow<T> row[COMP_K];
    float dtw[COMP_K];
};
// lane's COMP_K rows of the chunk that starts at sample j0 (rows past the ray's end are not touched and never used)
template <typename T>
__device__ __forceinline__ void load_chunk(const T* __restrict__ net, const float* __restrict__ coords, uint32_t base, uint32_t j0, uint32_t n,
                                           uint32_t lane, ChunkRaw<T>* c) {
#pragma unroll
    for (int q = 0; q < COMP_K; ++q) {
        const uint32_t j = j0 + COMP_K * lane + q;
        if (j < n) {
            load_row(net, (size_t)base + j, &c->row[q]);
            c->dtw[q] = __ldg(coords + ((size_t)base + j) * 7 + 3);
        } else {
            zero_row(&c->row[q]);                                    // evaluated unconditionally (no divergence), masked by alpha = 0
            c->dtw[q] = 0.f;
        }
    }
}
// forward over one ray: returns (all lanes) the composited colour WITHOUT background and the final transmittance
template <typename T>
__device__ __forceinline__ void composite_ray_fwd(uint32_t n, uint32_t base, const T* __restrict__ net, const float* __restrict__ coords,
                                                  uint32_t cascades, uint32_t lane, float rgb[3], float* T_final) {
    float carry = 1.f, acc[3] = {0.f, 0.f, 0.f};
    ChunkRaw<T> nxt;
    load_chunk<T>(net, coords, base, 0, n, lane, &nxt);
    for (uint32_t j0 = 0; j0 < n; j0 += 32 * COMP_K) {
        const ChunkRaw<T> cur = nxt;
        if (j0 + 32 * COMP_K < n) load_chunk<T>(net, coords, base, j0 + 32 * COMP_K, n, lane, &nxt);
        float a[COMP_K], c[COMP_K][3], p[COMP_K];                               // p[q] = prod_{r <= q} (1 - a[r]) over the lane's own samples
#pragma unroll
        for (int q = 0; q < COMP_K; ++q) {
            const Sample s = make_sample(row_f4(cur.row[q]), cur.dtw[q], cascades);
            a[q] = j0 + COMP_K * lane + q < n ? s.alpha : 0.f;
            c[q][0] = s.rgb[0]; c[q][1] = s.rgb[1]; c[q][2] = s.rgb[2];
            p[q] = q == 0 ? 1.f - a[q] : p[q - 1] * (1.f - a[q]);
        }
        const float incl = warp_incl_prod(p[COMP_K - 1], lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T_lane = carry * excl;                                      // transmittance in front of the lane's first sample
#pragma unroll
        for (int q = 0; q < COMP_K; ++q) {
            const float w = a[q] * (q == 0 ? T_lane : T_lane * p[q - 1]);
            acc[0] = __fmaf_rn(w, c[q][0], acc[0]); acc[1] = __fmaf_rn(w, c[q][1], acc[1]); acc[2] = __fmaf_rn(w, c[q][2], acc[2]);
        }
        carry *= __shfl_sync(0xffffffffu, incl, 31);
    }
    rgb[0] = warp_sum(acc[0]); rgb[1] = warp_sum(acc[1]); rgb[2] = warp_sum(acc[2]);
    *T_final = carry;
}

template <typename T>
__device__ __forceinline__ void composite_ray_bwd(uint32_t n, uint32_t base, const T* __restrict__ net, const float* __restrict__ coords,
                                                  const float lg[3], const float rr[3], float loss_scale, float l1, uint32_t cascades,
                                                  uint32_t lane, T* __restrict__ dnet) {
    float carry_T = 1.f, carry_S[3] = {0.f, 0.f, 0.f};
    for (uint32_t j0 = 0; j0 < n; j0 += 32 * COMP_K) {
        // no look-ahead here: the rows were read by the forward pass a moment ago (L1 / L2 hits, at most 8 rounds a ray), and the
        // 12 registers of a second chunk are what keeps a whole 4096-ray batch resident (<= 72 registers a thread)
        ChunkRaw<T> cur;
        load_chunk<T>(net, coords, base, j0, n, lane, &cur);
        float a[COMP_K], c[COMP_K][3], p[COMP_K], dt[COMP_K], sig[COMP_K];
#pragma unroll
        for (int q = 0; q < COMP_K; ++q) {
            const Sample s = make_sample(row_f4(cur.row[q]), cur.dtw[q], cascades);
            a[q] = j0 + COMP_K * lane + q < n ? s.alpha : 0.f;
            c[q][0] = s.rgb[0]; c[q][1] = s.rgb[1]; c[q][2] = s.rgb[2]; dt[q] = s.dt; sig[q] = s.sigma_raw;
            p[q] = q == 0 ? 1.f - a[q] : p[q - 1] * (1.f - a[q]);
        }
        const float incl = warp_incl_prod(p[COMP_K - 1], lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T_lane = carry_T * excl;
        float w[COMP_K], tot[3] = {0.f, 0.f, 0.f};                              // tot = colour accumulated over the lane's own samples
#pragma unroll
        for (int q = 0; q < COMP_K; ++q) {
            w[q] = a[q] * (q == 0 ? T_lane : T_lane * p[q - 1]);
#pragma unroll
            for (int k = 0; k < 3; ++k) tot[k] = __fmaf_rn(w[q], c[q][k], tot[k]);
        }
        float run[3], incl_S[3];                                                // run = colour accumulated up to (and then including) sample q
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            incl_S[k] = warp_incl_sum(tot[k], lane);
            float e = __shfl_up_sync(0xffffffffu, incl_S[k], 1);
            if (lane == 0) e = 0.f;
            run[k] = carry_S[k] + e;
        }
#pragma unroll
        for (int q = 0; q < COMP_K; ++q) {
            const uint32_t j = j0 + COMP_K * lane + q;
#pragma unroll
            for (int k = 0; k < 3; ++k) run[k] = __fmaf_rn(w[q], c[q][k], run[k]);         // rgb_ray2 including this sample
            if (j < n) {
                const float T_after = T_lane * p[q];                                        // T after this sample (calc_rgb.h:125)
                const float suffix[3] = {rr[0] - run[0], rr[1] - run[1], rr[2] - run[2]};
                float4 dl;
                dl.x = loss_scale * ((w[q] * lg[0]) * (c[q][0] * (1 - c[q][0])));           // calc_rgb.h:133-135 (l2 reg is 0 for Logistic)
                dl.y = loss_scale * ((w[q] * lg[1]) * (c[q][1] * (1 - c[q][1])));
                dl.z = loss_scale * ((w[q] * lg[2]) * (c[q][2] * (1 - c[q][2])));
                const float dd = __expf(fminf(fmaxf(sig[q], -15.0f), 15.0f));               // network_to_density_derivative
                const float dot = lg[0] * (T_after * c[q][0] - suffix[0]) +
                                  (lg[1] * (T_after * c[q][1] - suffix[1]) + lg[2] * (T_after * c[q][2] - suffix[2]));
                dl.w = loss_scale * (dd * (dt[q] * dot)) + (sig[q] < 0 ? -l1 : 0.0f);       // :137-139
                store_net<T>(dnet, (size_t)base + j, dl);
            }
        }
        carry_T *= __shfl_sync(0xffffffffu, incl, 31);
#pragma unroll
        for (int k = 0; k < 3; ++k) carry_S[k] += __shfl_sync(0xffffffffu, incl_S[k], 31);
    }
}

template <typename T, bool INFER>
__global__ void __launch_bounds__(256) composite_fwd_kernel(uint32_t n_rays, const T* __restrict__ net, const float* __restrict__ coords,
                                                            const uint32_t* __restrict__ numsteps_in, const uint32_t* __restrict__ numsteps_c,
                                                            const float* __restrict__ bg, uint32_t cascades, float* __restrict__ rgb_out,
                                                            float* __restrict__ alpha_out) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n_rays) return;
    const uint32_t n = numsteps_c[2 * i], base = numsteps_c[2 * i + 1];
    float r[3] = {0.f, 0.f, 0.f}, T_ = 1.f;
    if (n == 0) {
        if (!INFER) { r[0] = bg[3 * i]; r[1] = bg[3 * i + 1]; r[2] = bg[3 * i + 2]; }                // calc_rgb.h:35-39
    } else {
        composite_ray_fwd<T>(n, base, net, coords, cascades, lane, r, &T_);
        if (!INFER && n == numsteps_in[2 * i]) {                                                     // :68-71
            r[0] = __fmaf_rn(T_, bg[3 * i], r[0]); r[1] = __fmaf_rn(T_, bg[3 * i + 1], r[1]); r[2] = __fmaf_rn(T_, bg[3 * i + 2], r[2]);
        }
    }
    if (lane < 3) rgb_out[3 * i + lane] = r[lane];
    if (INFER && lane == 0) alpha_out[i] = (n == 0) ? 0.f : 1 - T_;
}

template <typename T>
__global__ void __launch_bounds__(256) composite_bwd_kernel(uint32_t n_rays, const T* __restrict__ net, const float* __restrict__ coords,
                                                            const uint32_t* __restrict__ numsteps_c, const float* __restrict__ loss_grad,
                                                            const float* __restrict__ rgb_ray, const float* __restrict__ mean, uint32_t cascades,
                                                            T* __restrict__ dnet) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n_rays) return;
    float loss_scale = 128;
    loss_scale /= n_rays;                                                                   // :100-101
    const float l1 = *mean < 0.01f ? 1e-4f : 0.0f;                                          // :112
    const float lg[3] = {loss_grad[3 * i], loss_grad[3 * i + 1], loss_grad[3 * i + 2]};
    const float rr[3] = {rgb_ray[3 * i], rgb_ray[3 * i + 1], rgb_ray[3 * i + 2]};
    composite_ray_bwd<T>(numsteps_c[2 * i], numsteps_c[2 * i + 1], net, coords, lg, rr, loss_scale, l1, cascades, lane, dnet);
}

// Fused training tail: composite forward, Huber gradient, composite backward -- one warp per ray.
__global__ void __launch_bounds__(128, 7) composite_loss_bwd_kernel(uint32_t n_rays, const __half* __restrict__ net, const float* __restrict__ coords,
                                                                 const uint32_t* __restrict__ numsteps_in, const uint32_t* __restrict__ numsteps_c,
                                                                 const float* __restrict__ bg, const float* __restrict__ target, float delta,
                                                                 const float* __restrict__ mean, uint32_t cascades, float* __restrict__ rgb_out,
                                                                 float* __restrict__ loss_out, __half* __restrict__ dnet, float reg_scale) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n_rays) return;
    const uint32_t n = numsteps_c[2 * i], base = numsteps_c[2 * i + 1];
    float T_ = 1.f, r[3] = {0.f, 0.f, 0.f};
    if (n == 0) { r[0] = bg[3 * i]; r[1] = bg[3 * i + 1]; r[2] = bg[3 * i + 2]; }
    else {
        composite_ray_fwd<__half>(n, base, net, coords, cascades, lane, r, &T_);
        if (n == numsteps_in[2 * i]) {
            r[0] = __fmaf_rn(T_, bg[3 * i], r[0]); r[1] = __fmaf_rn(T_, bg[3 * i + 1], r[1]); r[2] = __fmaf_rn(T_, bg[3 * i + 2], r[2]);
        }
    }
    float lg[3], loss = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {                                                           // huber_loss.py:11-14
        const float diff = r[k] - target[3 * i + k], rel = fabsf(diff);
        loss += rel > delta ? rel - 0.5f * delta : 0.5f / delta * rel * rel;
        lg[k] = rel > delta ? (diff > 0 ? 1.0f : -1.0f) : diff / delta;
    }
    if (lane < 3) rgb_out[3 * i + lane] = r[lane];
    if (loss_out && lane == 0) loss_out[i] = loss;
    float loss_scale = 128;
    loss_scale /= n_rays;
    // calc_rgb.h:112: the density regulariser is an absolute per-sample term, NOT scaled by 128 / n_rays.  Data-parallel shards
    // normalise by their local ray count and the exchange applies 1 / W: reg_scale = W keeps the regulariser what one GPU with the
    // global batch would add (without it a W-GPU run trains with 1/W of the sparsity pressure: -1.8 dB after 300 steps at W = 2)
    const float l1 = (*mean < 0.01f ? 1e-4f : 0.0f) * reg_scale;
    composite_ray_bwd<__half>(n, base, net, coords, lg, r, loss_scale, l1, cascades, lane, dnet);
}

}  // namespace

extern "C" {

uint64_t ngp_march_workspace_bytes(uint32_t n_rays) {
    // counts[n] | n_emit[n] | per ray: EmitRec[MARCH_EMIT_CAP]
    return (uint64_t)n_rays * (8 + MARCH_RAY_BYTES) + 1024;
}

int ngp_march(void* stream, uint32_t n_rays, float aabb_lo, float aabb_hi, uint32_t max_samples, const float* rays_o, const float* rays_d,
              const uint8_t* bitfield, float cone_angle, float near_distance, uint32_t cascades, int const_dt, uint64_t rng_state,
              uint64_t rng_inc, uint32_t* counters, uint32_t* ray_indices, uint32_t* numsteps, float* coords, void* workspace) {
    cudaStream_t s = (cudaStream_t)stream;
    NGP_REQUIRE(cascades >= 1 && cascades <= 8, "ngp_march: cascades out of range");
    NGP_CHECK_CUDA(cudaMemsetAsync(counters, 0, 8, s));                                     // ray_sampler.py:29
    if (n_rays == 0) return 0;
    const MarchCfg c = make_cfg(cascades, const_dt);
    const MarchRng mr{rng_state, rng_inc, 0u};
    uint32_t* counts = (uint32_t*)workspace;
    uint32_t* n_emit = counts + n_rays;
    uint8_t* ws = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(n_emit + n_rays) + 255) & ~(uintptr_t)255);
    const uint32_t blocks = (n_rays + MARCH_RAYS_PER_CTA - 1) / MARCH_RAYS_PER_CTA;   // two warps (producer, consumer) per ray
    march_count_kernel<<<blocks, 64 * MARCH_RAYS_PER_CTA, 0, s>>>(n_rays, aabb_lo, aabb_hi, rays_o, rays_d, bitfield, cone_angle, near_distance, c, mr,
                                                                 ws, counts, n_emit, ngp_err_flag());
    NGP_LAUNCH_CHECK();
    march_scan_kernel<<<1, 1024, 0, s>>>(n_rays, max_samples, counts, numsteps, ray_indices, counters);
    NGP_LAUNCH_CHECK();
    march_emit_kernel<<<n_rays, 128, 0, s>>>(n_rays, aabb_lo, aabb_hi, rays_o, rays_d, bitfield, cone_angle, near_distance, c, mr, numsteps, coords,
                                             ws, n_emit);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_compact(void* stream, uint32_t n_rays, uint32_t max_compacted, const float* coords_in, const uint32_t* numsteps_in, float* coords_out,
                uint32_t* numsteps_out, uint32_t* counters, int zero_fill) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n_rays == 0) { NGP_CHECK_CUDA(cudaMemsetAsync(counters, 0, 8, s)); return 0; }
    const int copy = coords_out != coords_in;   // aliased call: bookkeeping only (ray-ordered march output is already compact)
    compact_scan_kernel<<<1, 1024, 0, s>>>(n_rays, max_compacted, numsteps_in, numsteps_out, counters);
    NGP_LAUNCH_CHECK();
    if (copy) {
        compact_copy_kernel<<<(n_rays * 32 + 255) / 256, 256, 0, s>>>(n_rays, coords_in, numsteps_in, coords_out, numsteps_out);
        NGP_LAUNCH_CHECK();
    }
    if (zero_fill && copy) {
        zero_tail_kernel<<<ngp_num_sms(), 256, 0, s>>>(coords_out, counters, max_compacted);
        NGP_LAUNCH_CHECK();
    }
    return 0;
}

int ngp_composite_fwd(void* stream, uint32_t n_rays, const void* net_out, int dtype, const float* coords, const uint32_t* numsteps_in,
                      const uint32_t* numsteps_compacted, const float* bg, uint32_t cascades, float* rgb_out) {
    if (n_rays == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t blocks = (n_rays + 7) / 8;
    if (dtype == 1) composite_fwd_kernel<__half, false><<<blocks, 256, 0, s>>>(n_rays, (const __half*)net_out, coords, numsteps_in, numsteps_compacted, bg, cascades, rgb_out, nullptr);
    else if (dtype == 0) composite_fwd_kernel<float, false><<<blocks, 256, 0, s>>>(n_rays, (const float*)net_out, coords, numsteps_in, numsteps_compacted, bg, cascades, rgb_out, nullptr);
    else NGP_REQUIRE(false, "ngp_composite_fwd: bad dtype");
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_composite_infer(void* stream, uint32_t n_rays, const void* net_out, int dtype, const float* coords, const uint32_t* numsteps,
                        uint32_t cascades, float* rgb_out, float* alpha_out) {
    if (n_rays == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t blocks = (n_rays + 7) / 8;
    if (dtype == 1) composite_fwd_kernel<__half, true><<<blocks, 256, 0, s>>>(n_rays, (const __half*)net_out, coords, numsteps, numsteps, nullptr, cascades, rgb_out, alpha_out);
    else if (dtype == 0) composite_fwd_kernel<float, true><<<blocks, 256, 0, s>>>(n_rays, (const float*)net_out, coords, numsteps, numsteps, nullptr, cascades, rgb_out, alpha_out);
    else NGP_REQUIRE(false, "ngp_composite_infer: bad dtype");
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_composite_bwd(void* stream, uint32_t n_rays, uint32_t n_elements, const void* net_out, int dtype, const float* coords,
                      const uint32_t* numsteps_compacted, const float* loss_grad, const float* rgb_ray, const float* density_grid_mean,
                      uint32_t cascades, void* dnet_out) {
    NGP_REQUIRE(dtype == 0 || dtype == 1, "ngp_composite_bwd: bad dtype");
    cudaStream_t s = (cudaStream_t)stream;
    NGP_CHECK_CUDA(cudaMemsetAsync(dnet_out, 0, (size_t)n_elements * 4 * (dtype == 1 ? 2 : 4), s));   // DGS/calc_rgb.py:93
    if (n_rays == 0) return 0;
    const uint32_t blocks = (n_rays + 7) / 8;
    if (dtype == 1) composite_bwd_kernel<__half><<<blocks, 256, 0, s>>>(n_rays, (const __half*)net_out, coords, numsteps_compacted, loss_grad, rgb_ray, density_grid_mean, cascades, (__half*)dnet_out);
    else composite_bwd_kernel<float><<<blocks, 256, 0, s>>>(n_rays, (const float*)net_out, coords, numsteps_compacted, loss_grad, rgb_ray, density_grid_mean, cascades, (float*)dnet_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_elements, const void* net_out, const float* coords,
                           const uint32_t* numsteps_in, const uint32_t* numsteps_compacted, const float* bg, const float* target,
                           float huber_delta, const float* density_grid_mean, uint32_t cascades, float* rgb_out, float* loss_out, void* dnet_out,
                           float reg_scale) {
    (void)n_elements;   // rows not covered by a ray are never read downstream (the network backward is count-limited)
    if (n_rays == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    composite_loss_bwd_kernel<<<(n_rays + 3) / 4, 128, 0, s>>>(n_rays, (const __half*)net_out, coords, numsteps_in, numsteps_compacted, bg, target,
                                                               huber_delta, density_grid_mean, cascades, rgb_out, loss_out, (__half*)dnet_out, reg_scale);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
