// NGPNetworks.execute / .density and their backward as ONE kernel each (models/networks/ngp_network.py:77-89):
//   hash-grid gather (R2) -> density MLP 32->64->16 -> SH(dir) (R4) -> colour MLP 32->64->64->16 (R7) -> (N,4)
// Encoded features, SH features and all hidden activations stay in shared memory / registers; HBM sees only the
// 28 B coordinate, the 8 B output and (training) a 64 B encoded-feature row kept for backward.
//
// Backward reloads the 64 B encoded row, recomputes the MLP forward on the tensor cores (cheaper than storing
// 448 B of hidden activations per sample), runs the dgrad chain, accumulates all five weight gradients in registers
// across the CTA's tiles, and scatters dL/d(enc) into the hash-grid gradient (R3) without
// ever materialising dL/d(enc) in HBM.
//
// Roofline (DESIGN.md): forward is bound by the gather (524 B algorithmic per sample, L2-resident table);
// the tensor work is 20 480 flop/sample forward, 61 440 with dgrad+wgrad.
#include "mlp_tc.cuh"
#include "train_common.cuh"
#include <cstdlib>
#include <cstdio>
#include <mutex>
#include <vector>

int* ngp_err_flag();

namespace {
using namespace mlp;

// ---- shared-memory maps -------------------------------------------------------------------------------
// activation slab groups
constexpr uint32_t G_ENC = 0, G_HD = 4, G_RIN = 12, G_H1 = 16, G_H2F = 4 /* fwd: reuses hd */, G_H2B = 24;
constexpr uint32_t G_ENC1 = 24;   // forward kernel only: second (double-buffered) encoded-feature slab
struct SmemFwd {
    static constexpr uint32_t coords = 0;                         // two buffers of 128 x 7 f32 (3584 B each)
    static constexpr uint32_t act = 8192;                         // 28 groups: enc0 | hd/h2 | rin | h1 | enc1
    static constexpr uint32_t w0d = act + 28 * GB;
    static constexpr uint32_t woutd = w0d + 64 * 32 * 2;
    static constexpr uint32_t w0r = woutd + 16 * 64 * 2;
    static constexpr uint32_t w1r = w0r + 64 * 32 * 2;
    static constexpr uint32_t woutr = w1r + 64 * 64 * 2;
    static constexpr uint32_t levels = woutr + 16 * 64 * 2;
    static constexpr uint32_t total = levels + N_LEVELS * 32;
};
template <class S>
__device__ __forceinline__ void stage_all_weights(uint8_t* smem, const __half* wd, const __half* wr, uint32_t t) {
    stage_weights(smem + S::w0d, wd + WD_W0, 64, 32, t, 128);
    stage_weights(smem + S::woutd, wd + WD_WOUT, 16, 64, t, 128);
    if (wr) {
        stage_weights(smem + S::w0r, wr + WR_W0, 64, 32, t, 128);
        stage_weights(smem + S::w1r, wr + WR_W1, 64, 64, t, 128);
        stage_weights(smem + S::woutr, wr + WR_WOUT, 16, 64, t, 128);
    }
}

// Gather phase: thread (level = t&15, sub = t>>4) encodes the 16 CONSECUTIVE points 16*sub .. 16*sub+15 of the tile at its
// level.  Samples arrive ray-ordered, so consecutive points usually stay in the same grid cell at the coarser levels: the 8
// corner values are re-fetched only when the cell changes (run-length reuse).  The arithmetic per point is unchanged; the
// number of L1/L2 requests drops by the average run length (the gather is bound by request rate, not by bytes).
template <int STRIDE, int PTS>
__device__ __forceinline__ void gather_tile(const float* __restrict__ s_pos /* smem, STRIDE floats per row */, const NgpLevel& lv,
                                            const __half2* __restrict__ g, uint8_t* act, uint32_t g_enc, uint32_t level, uint32_t sub,
                                            __half* __restrict__ enc_save, uint32_t tile_row0, uint32_t n_live) {
    uint32_t cgx = 0xffffffffu, cgy = 0, cgz = 0;
    __half2 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = __float2half2_rn(0.f);
#pragma unroll 1
    for (int k = 0; k < PTS; ++k) {
        const uint32_t p = PTS * sub + k;
        const HashCell hc = hash_cell(lv, s_pos[p * STRIDE], s_pos[p * STRIDE + 1], s_pos[p * STRIDE + 2]);
        if (hc.gx != cgx || hc.gy != cgy || hc.gz != cgz) {
            cgx = hc.gx; cgy = hc.gy; cgz = hc.gz;
            uint32_t idx[8];
            hash_cell_indices(lv, cgx, cgy, cgz, idx);
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = __ldg(g + idx[c]);      // (pairing x-neighbours into 64-bit loads costs more issue slots than it saves here)
        }
        float w[8];
        hash_cell_weights(hc, w);
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float2 f = __half22float2(v[c]);
            a0 = fmaf(w[c], f.x, a0);
            a1 = fmaf(w[c], f.y, a1);
        }
        const __half2 r = __floats2half2_rn(a0, a1);
        *reinterpret_cast<__half2*>(act + (size_t)(g_enc + (level >> 2)) * GB + p * 16 + (level & 3) * 4) = r;
        if (enc_save && tile_row0 + p < n_live)
            *reinterpret_cast<__half2*>(enc_save + (size_t)(tile_row0 + p) * 32 + 2 * level) = r;
    }
}

// Forward chain of one warpgroup up to (and including) the colour net's last hidden layer.  Expects enc in ACT[G_ENC..+4) and,
// unless density_only, the SH features of the tile in ACT[G_RIN+2..+4).  Stores the fp16 density output h[0] of the thread's four
// fragment rows (64m + frag_row + 8h) in sig[2m + h] and leaves hd / rin / h1 / h2 in the slab.  bar_id: named barrier of the 128
// chain threads (0 = __syncthreads).
template <class S, uint32_t G_H2>
__device__ __forceinline__ void forward_chain(uint8_t* smem, uint32_t g_enc /* G_ENC or G_ENC1 */, uint32_t tw, bool density_only,
                                              uint32_t bar_id, uint16_t (&sig)[4]) {
    uint8_t* act = smem + S::act;
    const uint32_t smem_s = smem_u32(smem), act_s = smem_s + S::act;
    // density L0: enc(32) -> hd(64)
    layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<32, 64>(d, act_s, g_enc, smem_s + S::w0d, m); },
              [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_HD, m, tw); });
    operands_ready(bar_id, 128);
    // density L1: hd(64) -> h(16) = the first 16 colour-net inputs
    layer<16>([&](float (&d)[8], uint32_t m) { mma_fwd<64, 16>(d, act_s, G_HD, smem_s + S::woutd, m); },
              [&](const float (&d)[8], uint32_t m) {
                  sig[2 * m] = (uint16_t)(pack_half2(d[0], d[1]) & 0xFFFFu);
                  sig[2 * m + 1] = (uint16_t)(pack_half2(d[2], d[3]) & 0xFFFFu);
                  if (!density_only) frag_to_slab<16, false>(d, act, G_RIN, m, tw);
              });
    if (density_only) return;
    operands_ready(bar_id, 128);
    // colour L0: [h | sh](32) -> h1(64)
    layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<32, 64>(d, act_s, G_RIN, smem_s + S::w0r, m); },
              [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_H1, m, tw); });
    operands_ready(bar_id, 128);
    // colour L1: h1(64) -> h2(64)
    layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<64, 64>(d, act_s, G_H1, smem_s + S::w1r, m); },
              [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_H2, m, tw); });
    operands_ready(bar_id, 128);
}
// SH(dir) of row t -> ACT[G_RIN+2..+4), the last 16 colour-net inputs
__device__ __forceinline__ void sh_to_slab(uint8_t* act, const float* s_coords, uint32_t t) {
    float sh[16];
    sh4(s_coords[t * 7 + 4], s_coords[t * 7 + 5], s_coords[t * 7 + 6], sh);
    uint32_t p[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] = pack_half2(sh[2 * i], sh[2 * i + 1]);
    *reinterpret_cast<uint4*>(act + (G_RIN + 2) * GB + t * 16) = make_uint4(p[0], p[1], p[2], p[3]);
    *reinterpret_cast<uint4*>(act + (G_RIN + 3) * GB + t * 16) = make_uint4(p[4], p[5], p[6], p[7]);
}

// Warp-specialised forward: warps 4-7 ("gather") stage the coordinates of tile i+1 and encode them into one of two enc slabs while
// warps 0-3 ("chain") run the tensor-core MLP chain of tile i.  The gather is bound by the L1/L2 request rate, the chain by its
// serial stage latency; with both resident on the SM they overlap.  Hand-off through named barriers FULL[b] / EMPTY[b]
// (ids 2+b / 4+b, 256 threads: 128 arrive + 128 sync); the gather warps synchronise among themselves on barrier 6.
// Gather warps per CTA.  Measured on the lego stand-in: 4 warps x 16-point runs 104 us, 8 warps x 8-point runs 76 us per forward
// (the gather is instruction-latency bound with few warps; shorter runs cost a few more requests).
constexpr int FWD_GW = 8;
constexpr int FWD_THREADS = 128 + 32 * FWD_GW;

// Lattice mode (LATTICE, density only; extract_mesh.py:42-70): row r = (i*N + j)*N + k is the model position (i, j, k) / (N-1), made by
// the gather warps from the row index instead of staged from `coords`, and the epilogue writes float(int(max(sigma_raw, 0)))
// (extract_mesh.py:68) as fp32 into `out`.  The positions are IEEE quotients, so a coordinate buffer holding the same values gives the
// same sigma_raw bit for bit.
__device__ __forceinline__ float lattice_coord(uint32_t r, uint32_t axis, uint32_t n) {
    const uint32_t idx = axis == 0 ? r / (n * n) : axis == 1 ? (r / n) % n : r % n;
    return __fdiv_rn((float)idx, (float)(n - 1));
}

template <bool DENSITY_ONLY, bool LATTICE = false>
__global__ void __launch_bounds__(FWD_THREADS, 2)   // two CTAs per SM: <= 85 registers per thread
network_fwd_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const float* __restrict__ coords, const __half* __restrict__ grid,
                   const NgpLevel* __restrict__ levels, const __half* __restrict__ wd, const __half* __restrict__ wr,
                   __half* __restrict__ out, __half* __restrict__ enc_save, const __grid_constant__ NgpTensorMap enc_map, uint32_t enc_tma,
                   uint32_t lattice_n) {
    static_assert(DENSITY_ONLY || !LATTICE, "the lattice query is density only");
    // enc_tma: the encoded-feature rows kept for the backward pass leave the SM as four TMA tensor stores per tile, straight from the
    // slab the gather warps fill (one 8-column x 128-row box per feature group), instead of 16 four-byte global stores per row from the
    // gather warps -- which are the LSU-bound side of this kernel.  enc_save is then only the base address the tensor map was built for.
    extern __shared__ __align__(1024) uint8_t smem[];
    using S = SmemFwd;
    constexpr int CS = DENSITY_ONLY ? 3 : 7;
    const uint32_t t = threadIdx.x, warp = t >> 5;
    const bool is_chain = warp < 4;                                     // warps 0-3: the warpgroup that runs the MLP chain
    NgpLevel* s_lv = reinterpret_cast<NgpLevel*>(smem + S::levels);

    stage_weights(smem + S::w0d, wd + WD_W0, 64, 32, t, FWD_THREADS);
    stage_weights(smem + S::woutd, wd + WD_WOUT, 16, 64, t, FWD_THREADS);
    if (!DENSITY_ONLY) {
        stage_weights(smem + S::w0r, wr + WR_W0, 64, 32, t, FWD_THREADS);
        stage_weights(smem + S::w1r, wr + WR_W1, 64, 64, t, FWD_THREADS);
        stage_weights(smem + S::woutr, wr + WR_WOUT, 16, 64, t, FWD_THREADS);
    }
    if (t < N_LEVELS) s_lv[t] = levels[t];
    operands_ready(0, FWD_THREADS);
    const uint32_t n_live = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t ntiles = (n_live + ROWS - 1) / ROWS;

    if (is_chain) {
        uint8_t* act = smem + S::act;
        const uint32_t smem_s = smem_u32(smem), r0 = frag_row(t);
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1;
            const float* s_coords = reinterpret_cast<const float*>(smem + S::coords + buf * 3584);
            named_bar_sync(2 + buf, FWD_THREADS);                       // FULL[buf]: enc slab + coordinates of this tile are in smem
            if (!DENSITY_ONLY && enc_tma && warp == 0) {                 // the gather threads fenced their slab writes for the async proxy
                if (elect_one()) {
#pragma unroll
                    for (uint32_t g4 = 0; g4 < 4; ++g4)
                        tma_store_2d(&enc_map, 8 * g4, tile * ROWS, smem_s + S::act + ((buf ? G_ENC1 : G_ENC) + g4) * GB);
                    tma_store_commit();
                }
                __syncwarp();
            }
            if (!DENSITY_ONLY) sh_to_slab(act, s_coords, t);            // read by colour L0, after the chain's first barrier
            // forward_chain releases nothing itself: the enc slab is dead after layer 0, the coordinates after the SH features;
            // both are handed back together right after the chain (the gather runs a full tile ahead, so this is not on its path)
            uint16_t sig[4];
            forward_chain<S, G_H2F>(smem, buf ? G_ENC1 : G_ENC, t, DENSITY_ONLY, 1, sig);
            if (!DENSITY_ONLY && enc_tma && warp == 0) {                 // the tensor stores have read the slab before it is handed back
                if (elect_one()) tma_store_wait_read();
                __syncwarp();
            }
            if (tile + 2 * gridDim.x < ntiles) named_bar_arrive(4 + buf, FWD_THREADS);   // EMPTY[buf]
            if constexpr (DENSITY_ONLY) {
                if ((t & 3u) == 0) {
#pragma unroll
                    for (uint32_t i = 0; i < 4; ++i) {
                        const uint32_t row = tile * ROWS + 64 * (i >> 1) + r0 + 8 * (i & 1);
                        if (row >= n_live) continue;
                        if constexpr (LATTICE) reinterpret_cast<float*>(out)[row] = truncf(fmaxf(__half2float(__ushort_as_half(sig[i])), 0.f));
                        else reinterpret_cast<uint16_t*>(out)[row] = sig[i];
                    }
                }
            } else {
                layer<16>([&](float (&d)[8], uint32_t m) { mma_fwd<64, 16>(d, smem_s + S::act, G_H2F, smem_s + S::woutr, m); },
                          [&](const float (&d)[8], uint32_t m) {
#pragma unroll
                              for (uint32_t h = 0; h < 2; ++h) {
                                  const float c2 = __shfl_down_sync(0xffffffffu, d[2 * h], 1);   // column 2 sits in the next lane
                                  const uint32_t row = tile * ROWS + 64 * m + r0 + 8 * h;
                                  if ((t & 3u) == 0 && row < n_live) {
                                      uint2 o;
                                      o.x = pack_half2(d[2 * h], d[2 * h + 1]);
                                      o.y = (pack_half2(c2, 0.f) & 0xFFFFu) | ((uint32_t)sig[2 * m + h] << 16);
                                      reinterpret_cast<uint2*>(out)[row] = o;
                                  }
                              }
                          });
            }
            named_bar_sync(1, 128);                                      // this tile's wgmmas are done before the next tile's stores
        }
    } else {
        const uint32_t tg = t - 128, level = tg & 15, sub = tg >> 4;
        const NgpLevel lv = s_lv[level];
        const __half2* g = reinterpret_cast<const __half2*>(grid) + lv.offset;
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1, row0 = tile * ROWS;
            float* s_coords = reinterpret_cast<float*>(smem + S::coords + buf * 3584);
            if (it >= 2) named_bar_sync(4 + buf, FWD_THREADS);          // EMPTY[buf]: the chain of tile it-2 is done with this buffer
            for (uint32_t i = tg; i < ROWS * CS; i += 32 * FWD_GW) {     // stage the coordinate tile (coalesced)
                if constexpr (LATTICE) s_coords[i] = (row0 + i / CS < n_live) ? lattice_coord(row0 + i / CS, i % CS, lattice_n) : 0.f;
                else s_coords[i] = (row0 + i / CS < n_live) ? __ldg(coords + (size_t)row0 * CS + i) : 0.f;
            }
            named_bar_sync(6, 32 * FWD_GW);
            gather_tile<CS, 64 / FWD_GW>(s_coords, lv, g, smem + S::act, buf ? G_ENC1 : G_ENC, level, sub, (DENSITY_ONLY || enc_tma) ? nullptr : enc_save, row0,
                                         n_live);
            fence_proxy_async_smem();                           // the enc slab is read by the tensor core and the TMA (async proxy)
            named_bar_arrive(2 + buf, FWD_THREADS);                     // FULL[buf]
        }
    }
    if (!DENSITY_ONLY && enc_tma && warp == 0) {                         // shared memory must outlive the last tensor store
        if (elect_one()) tma_store_wait_all();
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward over 256 rows per stage (network_bwd256_kernel).
//
// The MLP chain is a strictly serial sequence of 10 stages per tile -- wgmma -> wait -> convert -> shared store -> barrier -- so two
// 128-row tiles move through the chain in lock step, one per warpgroup (warps 0-3: tile A, warps 4-7: tile B), and the weight
// gradients of both tiles accumulate into the same registers: each weight gradient is owned by one warpgroup, which contracts over
// the rows of both tiles (tile A's warpgroup: Woutr, W1r; tile B's: W0r, Woutd, W0d -- 40 accumulator registers each).  A barrier of
// the 256 chain threads ends every stage, so a weight-gradient wgmma of stage s may read the other tile's slabs written in stage s-1.
// Gradients rotate through buffers that died one stage earlier:
//     g_h2 -> GX (the one extra slab), g_h1 -> the h2 slab, dYd -> the dYr slab, g_hd -> the h1 slab,
// whose last reader (a weight-gradient wgmma) completed before the stage barrier the writing warpgroup passed.
// Warps: 0-7 MLP chain, 8-15 hash-grid scatter of the previous pair of tiles.
//
// Both gradient sums are independent of scheduling, so that a training run is reproducible: each CTA stores its weight-gradient sums
// in its own slot (layout [dwd | dwr]) and wgrad_reduce_kernel adds the slots in CTA order; the scatter adds into a 64-bit fixed-point
// copy of the hash-grid gradient (integer sums do not depend on their order) that grid_grad_flush_kernel rounds once into the fp16
// gradient and clears again -- or, after ngp_network_bwd_fx, the training sweep of optimizer.cu reads both straight from the slots
// and the scratch.  Without that scratch (see ngp_network_bwd) the kernel reduces straight into the outputs instead, with
// fp32 / f16x2 reductions whose rounding depends on their order.
constexpr uint32_t B3_G_GX = 32, B3_G_DY = 40, B3_G_DENC = 42, B3_GROUPS = 46;   // slab groups of one tile after the 32 activation groups
constexpr uint32_t B3_EPI_THREADS = 256, B3_SCATTER_WARPS = 8, B3_THREADS = B3_EPI_THREADS + 32 * B3_SCATTER_WARPS;
// scatter items: (level, run of B3_RUN consecutive rows of the pair), 16 levels x 12 runs, each walked by a group of 4 lanes
constexpr uint32_t B3_RUNS = 12, B3_ITEMS = 16 * B3_RUNS, B3_RUN = (2 * 128 + B3_RUNS - 1) / B3_RUNS;   // 22 rows
constexpr uint32_t B3_SCATTER_GROUPS = 32 * B3_SCATTER_WARPS / 4, B3_NI = B3_ITEMS / B3_SCATTER_GROUPS;   // 3 items per group
static_assert(B3_SCATTER_GROUPS % 16 == 0 && B3_ITEMS % B3_SCATTER_GROUPS == 0, "a lane group walks items of one level only, as many as every other group");
struct SmemBwd3 {
    static constexpr uint32_t coords = 0;                           // [tile][buf] 128 x 7 f32 (3584 B each)
    static constexpr uint32_t tile0 = coords + 4 * 3584;
    static constexpr uint32_t tile_stride = B3_GROUPS * GB;
    static constexpr uint32_t w0d = tile0 + 2 * tile_stride;
    static constexpr uint32_t woutd = w0d + 64 * 32 * 2;
    static constexpr uint32_t w0r = woutd + 16 * 64 * 2;
    static constexpr uint32_t w1r = w0r + 64 * 32 * 2;
    static constexpr uint32_t woutr = w1r + 64 * 64 * 2;
    static constexpr uint32_t levels = woutr + 16 * 64 * 2;
    static constexpr uint32_t dsig = levels + N_LEVELS * 32;        // [tile][128] fp16 dL/dsigma
    static constexpr uint32_t bar = dsig + 2 * ROWS * 2;            // [tile] mbarrier of the encoded-feature TMA loads
    static constexpr uint32_t total = bar + 16;
};
static_assert(SmemBwd3::total <= 227 * 1024, "backward CTA does not fit");
constexpr uint32_t B3_STAGE = 1, B3_FULL = 2, B3_EMPTY = 3;         // named barriers (4 + T: the 128 threads of tile T)

// a contribution to the fixed-point hash-grid gradient (train_common.cuh)
__device__ __forceinline__ void red_add_fx(unsigned long long* p, float v) {
    const long long q = __float2ll_rn(fminf(fmaxf(v, -65504.f), 65504.f) * FX_SCALE);
    if (q) asm volatile("red.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "l"((unsigned long long)q) : "memory");
}
// Feature f (= lane & 1) of entry idx of a level, held by this lane while its partner lane (lane ^ 1) holds the other feature of the
// same entry: into the fixed-point copy if the scratch holds the entry -- the two lanes' words are the 16 bytes of the entry, reduced
// by the same instruction -- and straight into the fp16 gradient otherwise, both features by the even lane.
__device__ __forceinline__ void red_add_entry_lane(unsigned long long* fx, uint32_t fx_live, __half2* gg, uint32_t idx, uint32_t f, float v) {
    if (idx < fx_live) {
        red_add_fx(fx + 2 * (size_t)idx + f, v);
    } else {
        const uint32_t lane = threadIdx.x & 31;
        const float o = __shfl_xor_sync(3u << (lane & 30), v, 1);
        if (!f) red_add_h2(gg + idx, v, o);
    }
}

// The MLP chain of tile T (one warpgroup) over all pairs of the CTA, then the flush of the weight gradients it owns.
template <uint32_t T>
__device__ __forceinline__ void bwd_chain(uint8_t* smem, uint32_t tid, uint32_t n_live, uint32_t npairs, const float* __restrict__ coords,
                                          const __half* __restrict__ enc_save, const __half* __restrict__ dout, float* __restrict__ w_part,
                                          float* __restrict__ dwd, float* __restrict__ dwr, int* __restrict__ err, uint32_t dbg, const NgpTensorMap* enc_map, uint32_t enc_tma) {
    using S = SmemBwd3;
    const uint32_t t = tid & 127, tq = (tid >> 5) & 3, r0 = frag_row(t);
    uint8_t* act = smem + S::tile0 + T * S::tile_stride;                // this tile's slabs
    const uint32_t smem_s = smem_u32(smem), a0 = smem_s + S::tile0, a1 = a0 + S::tile_stride, a_s = T ? a1 : a0;
    __half* s_dsig = reinterpret_cast<__half*>(smem + S::dsig) + T * ROWS;
    uint64_t* bar_t = reinterpret_cast<uint64_t*>(smem + S::bar) + T;
    const bool wg = !(dbg & 4);
    // zero-initialised: a CTA without a pair of tiles still stores its (empty) sums
    float acc_woutr[8] = {}, acc_w1r[32] = {};              // tile A's warpgroup: [64 in][16 out], [64 out][64 in]
    float acc_w0r[16] = {}, acc_woutd[8] = {}, acc_w0d[16] = {};   // tile B's warpgroup: [64 out][32 in], [64 in][16 out], [64 out][32 in]
    auto stage = [&]() { operands_ready(B3_STAGE, B3_EPI_THREADS); };
    float pf_c[7];
    uint4 pf_e[4];
    uint2 pf_d;
    auto prefetch = [&](uint32_t pair) {
        const uint32_t tile_ = 2 * pair + T, rr0 = tile_ * ROWS, r = rr0 + t;
        const bool ok = r < n_live;
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const uint32_t i = t + 128 * j;
            pf_c[j] = (rr0 + i / 7 < n_live) ? __ldg(coords + (size_t)rr0 * 7 + i) : 0.f;
        }
        if (!enc_tma) {
            const uint4* es = reinterpret_cast<const uint4*>(enc_save + (size_t)r * 32);
#pragma unroll
            for (int g = 0; g < 4; ++g) pf_e[g] = ok ? __ldg(es + g) : make_uint4(0, 0, 0, 0);
        }
        pf_d = ok ? __ldg(reinterpret_cast<const uint2*>(dout) + r) : make_uint2(0, 0);
    };
    if (blockIdx.x < npairs) prefetch(blockIdx.x);
    uint32_t it = 0, acc = 0;   // acc = 0 on the CTA's first pair: the weight-gradient accumulators are overwritten
    for (uint32_t pair = blockIdx.x; pair < npairs; pair += gridDim.x, ++it, acc = 1) {
        const uint32_t buf = it & 1;
        float* s_coords = reinterpret_cast<float*>(smem + S::coords + (2 * T + buf) * 3584);
        if (it >= 1) named_bar_sync(B3_STAGE, B3_EPI_THREADS);         // both warpgroups' wgmmas of the previous pair have read their slabs
#pragma unroll
        for (int j = 0; j < 7; ++j) s_coords[t + 128 * j] = pf_c[j];
        if (enc_tma) {
            // encoded-feature rows of this tile: four tensor loads (8-column x 128-row boxes = the four slab groups) by one thread
            if (tq == 0) {
                if (elect_one()) {
                    mbar_expect_tx(bar_t, ROWS * 64);
#pragma unroll
                    for (uint32_t g4 = 0; g4 < 4; ++g4)
                        tma_load_2d(smem_u32(act) + (G_ENC + g4) * GB, enc_map, 8 * g4, (2 * pair + T) * ROWS, bar_t);
                }
                __syncwarp();
            }
        } else {
#pragma unroll
            for (int g = 0; g < 4; ++g) *reinterpret_cast<uint4*>(act + (G_ENC + g) * GB + t * 16) = pf_e[g];
        }
        s_dsig[t] = __ushort_as_half((unsigned short)(pf_d.y >> 16));
        *reinterpret_cast<uint4*>(act + B3_G_DY * GB + t * 16) = make_uint4(pf_d.x, pf_d.y & 0xFFFFu, 0, 0);   // dYr: 3 colour gradients, K padded to 16
        *reinterpret_cast<uint4*>(act + (B3_G_DY + 1) * GB + t * 16) = make_uint4(0, 0, 0, 0);
        if (pair + gridDim.x < npairs) prefetch(pair + gridDim.x);     // in flight during the whole chain
        if (enc_tma) {
            if (!mbar_wait(bar_t, it & 1)) atomicExch(err, 4);
            if ((2 * pair + T) * ROWS + t >= n_live) {                  // rows past the live samples hold whatever an earlier step left: zero them
#pragma unroll
                for (int g = 0; g < 4; ++g) *reinterpret_cast<uint4*>(act + (G_ENC + g) * GB + t * 16) = make_uint4(0, 0, 0, 0);
            }
        }
        named_bar_sync(4 + T, 128);                                     // the SH features read other threads' coordinate words
        sh_to_slab(act, s_coords, t);
        stage();
        // F1 density L0: enc -> hd
        layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<32, 64>(d, a_s, G_ENC, smem_s + S::w0d, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_HD, m, t); });
        stage();
        // F2 density L1: hd -> h (16) = the first 16 colour-net inputs
        layer<16>([&](float (&d)[8], uint32_t m) { mma_fwd<64, 16>(d, a_s, G_HD, smem_s + S::woutd, m); },
                  [&](const float (&d)[8], uint32_t m) { frag_to_slab<16, false>(d, act, G_RIN, m, t); });
        stage();
        // F3 colour L0 -> h1 ; F4 colour L1 -> h2
        layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<32, 64>(d, a_s, G_RIN, smem_s + S::w0r, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_H1, m, t); });
        stage();
        layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<64, 64>(d, a_s, G_H1, smem_s + S::w1r, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_to_slab<64, true>(d, act, G_H2B, m, t); });
        stage();
        // B1: g_h2 = (dYr Woutr) . relu'(h2) -> GX ; Woutr [in][out] += h2^T dYr
        if (T == 0 && wg) { wgmma_fence(); mma_wgrad<16>(acc_woutr, a0, G_H2B, a0, B3_G_DY, acc); mma_wgrad<16>(acc_woutr, a1, G_H2B, a1, B3_G_DY, 1); }
        layer<64>([&](float (&d)[32], uint32_t m) { mma_dgrad<16, 64>(d, a_s, B3_G_DY, smem_s + S::woutr, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_dgrad_mask<64>(d, act, G_H2B, act, B3_G_GX, m, t); });
        stage();
        // B2: g_h1 = (g_h2 W1r) . relu'(h1) -> over h2 ; W1r [out][in] += g_h2^T h1
        if (T == 0 && wg) { wgmma_fence(); mma_wgrad<64>(acc_w1r, a0, B3_G_GX, a0, G_H1, acc); mma_wgrad<64>(acc_w1r, a1, B3_G_GX, a1, G_H1, 1); }
        layer<64>([&](float (&d)[32], uint32_t m) { mma_dgrad<64, 64>(d, a_s, B3_G_GX, smem_s + S::w1r, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_dgrad_mask<64>(d, act, G_H1, act, G_H2B, m, t); });
        stage();
        // B3: dYd = (g_h1 W0r)[:, 0..16) + dL/dsigma (ngp_network.py:83) -> over dYr (the other 16 columns of d_rin are dL/dSH, unused) ;
        //     W0r [out][in] += g_h1^T rin
        if (T == 1 && wg) { wgmma_fence(); mma_wgrad<32>(acc_w0r, a0, G_H2B, a0, G_RIN, acc); mma_wgrad<32>(acc_w0r, a1, G_H2B, a1, G_RIN, 1); }
        layer<16>([&](float (&d)[8], uint32_t m) { mma_dgrad<64, 16>(d, a_s, G_H2B, smem_s + S::w0r, m); },
                  [&](const float (&d)[8], uint32_t m) {
                      float v[8];
#pragma unroll
                      for (int i = 0; i < 8; ++i) v[i] = d[i];
                      if ((t & 3u) == 0) {                                // column 0 = dL/dsigma of rows r and r + 8
                          v[0] += __half2float(s_dsig[64 * m + r0]);
                          v[2] += __half2float(s_dsig[64 * m + r0 + 8]);
                      }
                      frag_to_slab<16, false>(v, act, B3_G_DY, m, t);
                  });
        stage();
        // B4: g_hd = (dYd Woutd) . relu'(hd) -> over h1 ; Woutd [in][out] += hd^T dYd
        if (T == 1 && wg) { wgmma_fence(); mma_wgrad<16>(acc_woutd, a0, G_HD, a0, B3_G_DY, acc); mma_wgrad<16>(acc_woutd, a1, G_HD, a1, B3_G_DY, 1); }
        layer<64>([&](float (&d)[32], uint32_t m) { mma_dgrad<16, 64>(d, a_s, B3_G_DY, smem_s + S::woutd, m); },
                  [&](const float (&d)[32], uint32_t m) { frag_dgrad_mask<64>(d, act, G_HD, act, G_H1, m, t); });
        stage();
        // B5: d_enc = g_hd W0d -> DENC (the scatter warps read the previous pair's until EMPTY) ; W0d [out][in] += g_hd^T enc
        if (T == 1 && wg) { wgmma_fence(); mma_wgrad<32>(acc_w0d, a0, G_H1, a0, G_ENC, acc); mma_wgrad<32>(acc_w0d, a1, G_H1, a1, G_ENC, 1); }
        if (it >= 1) named_bar_sync(B3_EMPTY, B3_EPI_THREADS + 32 * B3_SCATTER_WARPS);
        layer<32>([&](float (&d)[16], uint32_t m) { mma_dgrad<64, 32>(d, a_s, G_H1, smem_s + S::w0d, m); },
                  [&](const float (&d)[16], uint32_t m) { frag_to_slab<32, false>(d, act, B3_G_DENC, m, t); });
        named_bar_arrive(B3_FULL, B3_EPI_THREADS + 32 * B3_SCATTER_WARPS);   // dL/d(enc) and coords of this pair are ready
    }
    // the weight-gradient sums this warpgroup owns (colour Wout rows >= 3 stay zero, fully_fused_mlp.py:136): into the CTA's slot,
    // or without one added straight to the outputs
    if (!w_part) {
        if (!it) return;
        if (T == 0) {
            frag_red_add<16>(acc_woutr, dwr + WR_WOUT, 1, 64, 64, 3, t);
            frag_red_add<64>(acc_w1r, dwr + WR_W1, 64, 1, 64, 64, t);
        } else {
            frag_red_add<32>(acc_w0r, dwr + WR_W0, 32, 1, 64, 32, t);
            frag_red_add<16>(acc_woutd, dwd + WD_WOUT, 1, 64, 64, 16, t);
            frag_red_add<32>(acc_w0d, dwd + WD_W0, 32, 1, 64, 32, t);
        }
        return;
    }
    dwd = w_part + (size_t)blockIdx.x * W_PART;
    dwr = dwd + WD_N;
    if (T == 0) {
        frag_store<16>(acc_woutr, dwr + WR_WOUT, 1, 64, 3, t);
        frag_store<64>(acc_w1r, dwr + WR_W1, 64, 1, 64, t);
    } else {
        frag_store<32>(acc_w0r, dwr + WR_W0, 32, 1, 32, t);
        frag_store<16>(acc_woutd, dwd + WD_WOUT, 1, 64, 16, t);
        frag_store<32>(acc_w0d, dwd + WD_W0, 32, 1, 32, t);
    }
}

__global__ void __launch_bounds__(B3_THREADS, 1)
network_bwd256_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const float* __restrict__ coords, const __half* __restrict__ enc_save,
                      const NgpLevel* __restrict__ levels, const __half* __restrict__ wd, const __half* __restrict__ wr,
                      const __half* __restrict__ dout, __half* __restrict__ grid_grad, float* __restrict__ dwd, float* __restrict__ dwr,
                      unsigned long long* __restrict__ grid_fx, uint32_t fx_entries, float* __restrict__ w_part,
                      int* __restrict__ err, uint32_t dbg, const __grid_constant__ NgpTensorMap enc_map, uint32_t enc_tma) {
    extern __shared__ __align__(1024) uint8_t smem[];
    using S = SmemBwd3;
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    uint64_t* bar_t = reinterpret_cast<uint64_t*>(smem + S::bar);
    NgpLevel* s_lv = reinterpret_cast<NgpLevel*>(smem + S::levels);

    stage_weights(smem + S::w0d, wd + WD_W0, 64, 32, tid, B3_THREADS);
    stage_weights(smem + S::woutd, wd + WD_WOUT, 16, 64, tid, B3_THREADS);
    stage_weights(smem + S::w0r, wr + WR_W0, 64, 32, tid, B3_THREADS);
    stage_weights(smem + S::w1r, wr + WR_W1, 64, 64, tid, B3_THREADS);
    stage_weights(smem + S::woutr, wr + WR_WOUT, 16, 64, tid, B3_THREADS);
    if (tid < N_LEVELS) s_lv[tid] = levels[tid];
    // zero both tiles once: dYr columns 4..15 are never rewritten, and 64-feature weight-gradient operands run past their slab
    for (uint32_t i = tid; i < 2 * S::tile_stride / 16; i += B3_THREADS) *reinterpret_cast<uint4*>(smem + S::tile0 + i * 16) = make_uint4(0, 0, 0, 0);
    if (tid == 0) { mbar_init(bar_t, 1); mbar_init(bar_t + 1, 1); fence_mbar_init(); }
    operands_ready(0, B3_THREADS);
    const uint32_t n_live = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t ntiles = (n_live + ROWS - 1) / ROWS, npairs = (ntiles + 1) / 2;

    if (warp < 4) {
        bwd_chain<0>(smem, tid, n_live, npairs, coords, enc_save, dout, w_part, dwd, dwr, err, dbg, &enc_map, enc_tma);
    } else if (warp < 8) {
        bwd_chain<1>(smem, tid, n_live, npairs, coords, enc_save, dout, w_part, dwd, dwr, err, dbg, &enc_map, enc_tma);
    } else {
        // ------------------------------------------------------------------ scatter (HashEncode.h:339-347) of the pair's 256 rows
        // Item (level, sub) is a run of B3_RUN consecutive samples of one level, walked by a group of 4 adjacent lanes: every lane of the
        // group reads the same rows, skips the same rows and sees the same cell changes, and accumulates its own 4 (corner, feature) slots
        // in fp32 registers while the grid cell stays the same.  Lane bit 0 is the feature f, bit 1 picks the corner 2j + h of each
        // x-neighbour pair (2j, 2j + 1).  At a cell change slot j of the 4 lanes is reduced by one instruction: both features of both
        // x-neighbours, 32 bytes of the fixed-point copy, which are one aligned sector whenever the pair's entries are 2k and 2k + 1.
        const uint32_t ts = tid - B3_EPI_THREADS, grp = ts >> 2, f = ts & 1, h = (ts >> 1) & 1;
        const uint32_t level = grp & 15;                                         // item = grp + k * B3_SCATTER_GROUPS: level = item & 15
        const NgpLevel lv = s_lv[level];
        unsigned long long* fx = grid_fx + 2 * (size_t)lv.offset;
        const uint32_t fx_live = fx_entries > lv.offset ? fx_entries - lv.offset : 0u;     // entries of this level the scratch holds
        __half2* gg = reinterpret_cast<__half2*>(grid_grad) + lv.offset;
        // The group's B3_NI items (grp + i * B3_SCATTER_GROUPS) are walked side by side, row k of each in the same iteration: their
        // shared-memory reads and cell arithmetic are independent, so they overlap instead of adding up.  Each item still sees its rows
        // in order, so its run sums are the same; only the order of the (integer, order-free) reductions across items changes.
        uint32_t it = 0;
        for (uint32_t pair = blockIdx.x; pair < npairs; pair += gridDim.x, ++it) {
            const uint32_t buf = it & 1;
            named_bar_sync(B3_FULL, B3_EPI_THREADS + 32 * B3_SCATTER_WARPS);
            uint32_t cgx[B3_NI], cgy[B3_NI], cgz[B3_NI], idx[B3_NI][4];
            float acc[B3_NI][4];
            bool live[B3_NI], dirty[B3_NI];
#pragma unroll
            for (uint32_t i = 0; i < B3_NI; ++i) { cgx[i] = 0xffffffffu; cgy[i] = cgz[i] = 0; live[i] = !(dbg & 2); dirty[i] = false; }
#pragma unroll 1
            for (uint32_t k = 0; k < B3_RUN; ++k) {
                float2 df[B3_NI];
                HashCell hc[B3_NI];
#pragma unroll
                for (uint32_t i = 0; i < B3_NI; ++i) {
                    const uint32_t r = B3_RUN * ((grp + i * B3_SCATTER_GROUPS) >> 4) + k;   // row of the pair: tile r >> 7, row r & 127
                    live[i] = live[i] && r < 2 * ROWS && 2 * pair * ROWS + r < n_live;        // rows past the pair or the live rows end the run
                    const uint32_t rc = min(r, 2 * ROWS - 1), T = rc >> 7, p = rc & 127;       // read in bounds either way
                    const uint8_t* denc = smem + S::tile0 + T * S::tile_stride + B3_G_DENC * GB;
                    const float* s_coords = reinterpret_cast<const float*>(smem + S::coords + (2 * T + buf) * 3584);
                    df[i] = __half22float2(*reinterpret_cast<const __half2*>(denc + (size_t)(level >> 2) * GB + p * 16 + (level & 3) * 4));
                    hc[i] = hash_cell(lv, s_coords[p * 7], s_coords[p * 7 + 1], s_coords[p * 7 + 2]);
                }
#pragma unroll
                for (uint32_t i = 0; i < B3_NI; ++i) {
                    if (!live[i] || (df[i].x == 0.f && df[i].y == 0.f)) continue;
                    if (hc[i].gx != cgx[i] || hc[i].gy != cgy[i] || hc[i].gz != cgz[i]) {
                        if (dirty[i] && !(dbg & 1)) {
#pragma unroll
                            for (uint32_t j = 0; j < 4; ++j) red_add_entry_lane(fx, fx_live, gg, idx[i][j], f, acc[i][j]);
                        }
                        cgx[i] = hc[i].gx; cgy[i] = hc[i].gy; cgz[i] = hc[i].gz;
                        uint32_t ci[8];
                        hash_cell_indices(lv, cgx[i], cgy[i], cgz[i], ci);
#pragma unroll
                        for (uint32_t j = 0; j < 4; ++j) { idx[i][j] = h ? ci[2 * j + 1] : ci[2 * j]; acc[i][j] = 0.f; }
                        dirty[i] = true;
                    }
                    // weight of corner 2j + h, formed as hash_cell_weights forms it, so that every per-run sum stays bit for bit the same
                    const float dv = f ? df[i].y : df[i].x;
                    const float wx = h ? hc[i].fx : 1.0f - hc[i].fx;
                    const float wy[2] = {1.0f - hc[i].fy, hc[i].fy}, wz[2] = {1.0f - hc[i].fz, hc[i].fz};
#pragma unroll
                    for (uint32_t j = 0; j < 4; ++j) acc[i][j] = fmaf(dv, (1.0f * wx) * wy[j & 1] * wz[j >> 1], acc[i][j]);
                }
            }
#pragma unroll
            for (uint32_t i = 0; i < B3_NI; ++i) {
                if (dirty[i] && !(dbg & 1)) {
#pragma unroll
                    for (uint32_t j = 0; j < 4; ++j) red_add_entry_lane(fx, fx_live, gg, idx[i][j], f, acc[i][j]);
                }
            }
            if (pair + gridDim.x < npairs) named_bar_arrive(B3_EMPTY, B3_EPI_THREADS + 32 * B3_SCATTER_WARPS);
        }
    }
}

// dwd / dwr += the CTAs' weight-gradient sums, added in CTA order
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, uint32_t nparts, float* __restrict__ dwd, float* __restrict__ dwr) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (uint32_t)W_PART) return;
    // four running sums over slots k = 0, 1, 2, 3 (mod 4) keep 16 loads in flight; the order of the additions is fixed
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
    const float sum = (a0 + a1) + (a2 + a3);
    if (e < (uint32_t)WD_N) dwd[e] += sum; else dwr[e - WD_N] += sum;
}

// grid_grad += the fixed-point sums (one fp16 rounding per feature), and the touched fixed-point entries back to zero.  The level table
// gives the number of entries; entries beyond the scratch were reduced into grid_grad directly.
__global__ void grid_grad_flush_kernel(const NgpLevel* __restrict__ levels, uint32_t fx_entries, longlong2* __restrict__ fx,
                                       __half2* __restrict__ grid_grad) {
    const uint32_t n = min(levels[N_LEVELS - 1].offset + levels[N_LEVELS - 1].size, fx_entries);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const longlong2 q = fx[i];
        if (q.x | q.y) {
            float2 g = __half22float2(grid_grad[i]);
            g.x += __ll2float_rn(q.x) * FX_INV;
            g.y += __ll2float_rn(q.y) * FX_INV;
            grid_grad[i] = __floats2half2_rn(g.x, g.y);
            fx[i] = make_longlong2(0, 0);
        }
    }
}

// Scratch of ngp_network_bwd, one per (device, stream) so that calls on different streams never share it: the fixed-point gradient,
// sized from the level table when a table is first seen on that stream, and the per-CTA weight-gradient slots.
struct BwdScratch {
    int dev = -1;
    cudaStream_t stream = nullptr;
    const void* levels = nullptr;
    uint32_t fx_entries = 0;
    unsigned long long* fx = nullptr;
    float* part = nullptr;
};
std::mutex g_scratch_mu;
std::vector<BwdScratch*> g_scratch;

// The scratch for this call, or nullptr (the call then reduces straight into its outputs) when it cannot be set up: inside graph
// capture, where nothing may be allocated or read back.  A table seen for the first time costs one read-back of its last level.
int bwd_scratch(cudaStream_t s, const void* levels_dev, BwdScratch** out) {
    *out = nullptr;
    int dev = 0;
    NGP_CHECK_CUDA(cudaGetDevice(&dev));
    BwdScratch* b = nullptr;
    {
        std::lock_guard<std::mutex> lock(g_scratch_mu);
        for (BwdScratch* e : g_scratch)
            if (e->dev == dev && e->stream == s) b = e;
        if (!b) {
            b = new BwdScratch;
            b->dev = dev;
            b->stream = s;
            g_scratch.push_back(b);
        }
    }
    if (b->levels == levels_dev && b->part) { *out = b; return 0; }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    NGP_CHECK_CUDA(cudaStreamIsCapturing(s, &cap));
    if (cap != cudaStreamCaptureStatusNone) return 0;
    NgpLevel last;
    NGP_CHECK_CUDA(cudaMemcpyAsync(&last, reinterpret_cast<const NgpLevel*>(levels_dev) + N_LEVELS - 1, sizeof(last), cudaMemcpyDeviceToHost, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    const uint32_t entries = last.offset + last.size;
    if (entries > b->fx_entries) {
        if (b->fx) NGP_CHECK_CUDA(cudaFree(b->fx));
        b->fx = nullptr;
        b->fx_entries = 0;
        NGP_CHECK_CUDA(cudaMalloc(&b->fx, sizeof(unsigned long long) * 2 * (size_t)entries));
        NGP_CHECK_CUDA(cudaMemset(b->fx, 0, sizeof(unsigned long long) * 2 * (size_t)entries));
        b->fx_entries = entries;
    }
    if (!b->part) NGP_CHECK_CUDA(cudaMalloc(&b->part, sizeof(float) * W_PART * (size_t)ngp_num_sms()));
    b->levels = levels_dev;
    *out = b;
    return 0;
}

// One launch of network_bwd256_kernel: with fx / w_part into the fixed-point scratch and the per-CTA slots, without them straight
// into grid_grad / dwd / dwr.
int bwd_launch(cudaStream_t s, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* enc_save, const void* levels_dev,
               const void* w_density, const void* w_rgb, const void* dout, void* grid_grad, float* dw_density, float* dw_rgb,
               unsigned long long* fx, uint32_t fx_entries, float* w_part) {
    // timing experiments only (results are wrong with any bit set): 1 = no atomics, 2 = no scatter, 4 = no weight-gradient MMAs
    static const uint32_t dbg = getenv("NGP_BWD_DEBUG") ? (uint32_t)atoi(getenv("NGP_BWD_DEBUG")) : 0u;
    if (ngp_first_use((const void*)network_bwd256_kernel)) NGP_CHECK_CUDA(cudaFuncSetAttribute(network_bwd256_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmemBwd3::total));
    NgpTensorMap enc_map{};
    static const bool no_tma = getenv("NGP_NO_TMA") != nullptr;           // A/B switch
    const uint32_t enc_tma = (!no_tma && ngp_make_rows32_tensormap(&enc_map, enc_save, n_max)) ? 1u : 0u;
    network_bwd256_kernel<<<bwd_ctas(n_max), B3_THREADS, SmemBwd3::total, s>>>(n_max, n_dev, coords, (const __half*)enc_save, (const NgpLevel*)levels_dev,
                                                                              (const __half*)w_density, (const __half*)w_rgb, (const __half*)dout,
                                                                              (__half*)grid_grad, dw_density, dw_rgb, fx, fx_entries, w_part,
                                                                              ngp_err_flag(), dbg, enc_map, enc_tma);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" {

int ngp_network_fwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* grid, const void* levels_dev,
                    const void* w_density, const void* w_rgb, void* out, void* enc_save) {
    if (n_max == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    if (ngp_first_use((const void*)network_fwd_kernel<false>)) NGP_CHECK_CUDA(cudaFuncSetAttribute(network_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmemFwd::total));
    const uint32_t ntiles = (n_max + ROWS - 1) / ROWS;
    const uint32_t grid_dim = min(ntiles, (uint32_t)ngp_num_sms() * 2u);
    NgpTensorMap enc_map{};
    static const bool no_tma = getenv("NGP_NO_TMA") != nullptr;           // A/B switch
    const uint32_t enc_tma = (!no_tma && enc_save && ngp_make_rows32_tensormap(&enc_map, enc_save, n_max)) ? 1u : 0u;
    network_fwd_kernel<false><<<grid_dim, FWD_THREADS, SmemFwd::total, s>>>(n_max, n_dev, coords, (const __half*)grid, (const NgpLevel*)levels_dev,
                                                                   (const __half*)w_density, (const __half*)w_rgb, (__half*)out,
                                                                   (__half*)enc_save, enc_map, enc_tma, 0u);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_density_fwd(void* stream, uint32_t n, const float* pos, const void* grid, const void* levels_dev, const void* w_density, void* sigma_out) {
    if (n == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    if (ngp_first_use((const void*)network_fwd_kernel<true>)) NGP_CHECK_CUDA(cudaFuncSetAttribute(network_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmemFwd::total));
    const uint32_t ntiles = (n + ROWS - 1) / ROWS;
    const uint32_t grid_dim = min(ntiles, (uint32_t)ngp_num_sms() * 2u);
    network_fwd_kernel<true><<<grid_dim, FWD_THREADS, SmemFwd::total, s>>>(n, nullptr, pos, (const __half*)grid, (const NgpLevel*)levels_dev,
                                                                  (const __half*)w_density, nullptr, (__half*)sigma_out, nullptr, NgpTensorMap{}, 0u, 0u);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_density_lattice(void* stream, uint32_t n, const void* grid, const void* levels_dev, const void* w_density, float* field_out) {
    NGP_REQUIRE(n >= 2 && n <= 1024, "ngp_density_lattice: resolution n must be in [2, 1024], got " + std::to_string(n));
    cudaStream_t s = (cudaStream_t)stream;
    if (ngp_first_use((const void*)network_fwd_kernel<true, true>))
        NGP_CHECK_CUDA(cudaFuncSetAttribute(network_fwd_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmemFwd::total));
    const uint32_t n3 = n * n * n, ntiles = (n3 + ROWS - 1) / ROWS;
    const uint32_t grid_dim = min(ntiles, (uint32_t)ngp_num_sms() * 2u);
    network_fwd_kernel<true, true><<<grid_dim, FWD_THREADS, SmemFwd::total, s>>>(n3, nullptr, nullptr, (const __half*)grid, (const NgpLevel*)levels_dev,
                                                                                (const __half*)w_density, nullptr, reinterpret_cast<__half*>(field_out),
                                                                                nullptr, NgpTensorMap{}, 0u, n);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_network_bwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* enc_save, const void* levels_dev,
                    const void* w_density, const void* w_rgb, const void* dout, void* grid_grad, float* dw_density, float* dw_rgb) {
    if (n_max == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    BwdScratch* b = nullptr;
    if (int rc = bwd_scratch(s, levels_dev, &b)) return rc;
    if (int rc = bwd_launch(s, n_max, n_dev, coords, enc_save, levels_dev, w_density, w_rgb, dout, grid_grad, dw_density, dw_rgb, b ? b->fx : nullptr,
                            b ? b->fx_entries : 0u, b ? b->part : nullptr))
        return rc;
    if (b) {
        wgrad_reduce_kernel<<<(W_PART + 255) / 256, 256, 0, s>>>(b->part, bwd_ctas(n_max), dw_density, dw_rgb);
        NGP_LAUNCH_CHECK();
        grid_grad_flush_kernel<<<ngp_num_sms() * 8, 256, 0, s>>>((const NgpLevel*)levels_dev, b->fx_entries, reinterpret_cast<longlong2*>(b->fx),
                                                                 (__half2*)grid_grad);
        NGP_LAUNCH_CHECK();
    }
    return 0;
}

int ngp_network_bwd_fx_bytes(uint64_t n_entries, uint64_t* fx_bytes, uint64_t* part_bytes) {
    *fx_bytes = 16 * n_entries;
    *part_bytes = sizeof(float) * W_PART * (uint64_t)ngp_num_sms();
    return 0;
}

int ngp_network_bwd_fx(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* enc_save, const void* levels_dev,
                       const void* w_density, const void* w_rgb, const void* dout, uint32_t n_entries, void* fx, uint64_t fx_bytes,
                       float* w_part, uint64_t part_bytes) {
    // every entry must be held by the scratch: the kernel's fallback for the others would reduce into a gradient this call has not got
    NGP_REQUIRE(fx != nullptr && fx_bytes >= 16 * (uint64_t)n_entries, "ngp_network_bwd_fx: the fixed-point scratch must hold 16 bytes per table entry");
    NGP_REQUIRE(w_part != nullptr && part_bytes >= sizeof(float) * W_PART * (uint64_t)ngp_num_sms(),
                "ngp_network_bwd_fx: the weight-gradient slots are smaller than ngp_network_bwd_fx_bytes gives");
    if (n_max == 0) return 0;
    return bwd_launch((cudaStream_t)stream, n_max, n_dev, coords, enc_save, levels_dev, w_density, w_rgb, dout, nullptr, nullptr, nullptr,
                      (unsigned long long*)fx, n_entries, w_part);
}

}  // extern "C"
