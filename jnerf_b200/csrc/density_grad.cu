// ngp_density_grad: the gradient of the fused NGP density output h0 (sigma_raw, before exp) with respect to the warped position, for
// the renderer's normal maps (DESIGN.md section 4, "Rendering").  Per row, with enc the fp16 hash-grid encoding and hd = W0d enc:
//     grad = sum over levels l of J_l^T g_enc[2l .. 2l+2),   g_enc = W0d^T (mask .* Woutd[0, :]),   mask = hd > 0,
// J_l the 2x3 derivative of level l's two features, scale_l * sum_c v_c dw_c/dfrac over the cell's 8 corner values.
// The layout is the fused forward's (fused_net.cu): gather warps encode tile i+1 into an fp16 slab, exactly as gather_tile does, and
// also write J to shared memory, while the chain warpgroup forms density L0 of tile i with the forward's own wgmma (so the mask is the
// forward's, bit for bit) and then the rest in fp32 on the CUDA cores: about 2.2 k FMA a row against the gather's 128 corner loads.
#include "mlp_tc.cuh"
#include "train_common.cuh"

namespace {
using namespace mlp;

// One CTA per SM (the two J buffers take 97 KB), so twice the forward's gather warps per CTA: the same 16 gather warps per SM.
constexpr int DG_GW = 16;
constexpr int DG_THREADS = 128 + 32 * DG_GW;
constexpr uint32_t DG_PTS = 128 / (2 * DG_GW);         // consecutive points per gather thread and level
constexpr uint32_t DG_LD = ROWS + 1;                   // floats between the planes of J and u: rows of one plane in consecutive banks,
                                                       // the 16 levels' planes of one row in distinct banks
constexpr uint32_t align1k(uint32_t x) { return (x + 1023u) & ~1023u; }
struct SmemGrad {
    static constexpr uint32_t coords = 0;                               // two buffers of 128 x 7 f32 (3584 B each)
    static constexpr uint32_t enc = 8192;                               // two fp16 encoding slabs of 4 groups each
    static constexpr uint32_t jac = enc + 8 * GB;                       // two buffers of 96 planes: J[level][feature][axis][row]
    static constexpr uint32_t jac_bytes = 96 * DG_LD * 4;
    static constexpr uint32_t u = jac + 2 * jac_bytes;                  // 64 planes: u[hidden][row] = mask .* Woutd[0, hidden]
    static constexpr uint32_t w0d = align1k(u + 64 * DG_LD * 4);        // W0d staged for the wgmma
    static constexpr uint32_t w0f = w0d + 64 * 32 * 2;                  // W0d in fp32, row-major [hidden][input]
    static constexpr uint32_t levels = w0f + 64 * 32 * 4;
    static constexpr uint32_t total = levels + N_LEVELS * 32;
};
static_assert(SmemGrad::total <= 227 * 1024, "density-gradient CTA does not fit");

// gather_tile of fused_net.cu (the same encoding, bit for bit) plus the Jacobian of the level's two features at each point.
__device__ __forceinline__ void gather_tile_jac(const float* __restrict__ s_pos, const NgpLevel& lv, const __half2* __restrict__ g, uint8_t* act,
                                                uint32_t g_enc, float* __restrict__ jac, uint32_t level, uint32_t sub) {
    uint32_t cgx = 0xffffffffu, cgy = 0, cgz = 0;
    __half2 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = __float2half2_rn(0.f);
#pragma unroll 1
    for (uint32_t k = 0; k < DG_PTS; ++k) {
        const uint32_t p = DG_PTS * sub + k;
        const HashCell hc = hash_cell(lv, s_pos[p * 7], s_pos[p * 7 + 1], s_pos[p * 7 + 2]);
        if (hc.gx != cgx || hc.gy != cgy || hc.gz != cgz) {
            cgx = hc.gx; cgy = hc.gy; cgz = hc.gz;
            uint32_t idx[8];
            hash_cell_indices(lv, cgx, cgy, cgz, idx);
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = __ldg(g + idx[c]);
        }
        float w[8];
        hash_cell_weights(hc, w);
        const float wx[2] = {1.0f - hc.fx, hc.fx}, wy[2] = {1.0f - hc.fy, hc.fy}, wz[2] = {1.0f - hc.fz, hc.fz};
        float a0 = 0.f, a1 = 0.f, j[2][3] = {};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float2 f = __half22float2(v[c]);
            a0 = fmaf(w[c], f.x, a0);
            a1 = fmaf(w[c], f.y, a1);
            // dw_c / dfrac: the weight with its own axis' factor replaced by -1 (corner at 0) or +1 (corner at 1)
            const float dx = wy[(c >> 1) & 1] * wz[c >> 2], dy = wx[c & 1] * wz[c >> 2], dz = wx[c & 1] * wy[(c >> 1) & 1];
            const float d[3] = {(c & 1) ? dx : -dx, (c & 2) ? dy : -dy, (c & 4) ? dz : -dz};
#pragma unroll
            for (int a = 0; a < 3; ++a) { j[0][a] = fmaf(d[a], f.x, j[0][a]); j[1][a] = fmaf(d[a], f.y, j[1][a]); }
        }
        *reinterpret_cast<__half2*>(act + (size_t)(g_enc + (level >> 2)) * GB + p * 16 + (level & 3) * 4) = __floats2half2_rn(a0, a1);
#pragma unroll
        for (int f = 0; f < 2; ++f)
#pragma unroll
            for (int a = 0; a < 3; ++a) jac[(6 * level + 3 * f + a) * DG_LD + p] = lv.scale * j[f][a];
    }
}

__global__ void __launch_bounds__(DG_THREADS, 1)
density_grad_kernel(uint32_t n_max, const uint32_t* __restrict__ n_dev, const float* __restrict__ coords, const __half* __restrict__ grid,
                    const NgpLevel* __restrict__ levels, const __half* __restrict__ wd, float* __restrict__ grad_out) {
    extern __shared__ __align__(1024) uint8_t smem[];
    using S = SmemGrad;
    const uint32_t t = threadIdx.x, warp = t >> 5;
    NgpLevel* s_lv = reinterpret_cast<NgpLevel*>(smem + S::levels);
    float* s_w0 = reinterpret_cast<float*>(smem + S::w0f);

    stage_weights(smem + S::w0d, wd + WD_W0, 64, 32, t, DG_THREADS);
    for (uint32_t i = t; i < 64 * 32; i += DG_THREADS) s_w0[i] = __half2float(wd[WD_W0 + i]);
    if (t < N_LEVELS) s_lv[t] = levels[t];
    operands_ready(0, DG_THREADS);
    const uint32_t n_live = n_dev ? min(*n_dev, n_max) : n_max;
    const uint32_t ntiles = (n_live + ROWS - 1) / ROWS;

    if (warp < 4) {                                                     // chain: L0 mask, g_enc, J^T g_enc of row t
        const uint32_t smem_s = smem_u32(smem), r0 = frag_row(t), cb = 2u * (t & 3u);
        float* s_u = reinterpret_cast<float*>(smem + S::u);
        float wo[16];                                                   // Woutd[0, col] of the thread's fragment columns 8c + cb + j
#pragma unroll
        for (uint32_t c = 0; c < 8; ++c)
#pragma unroll
            for (uint32_t j = 0; j < 2; ++j) wo[2 * c + j] = __half2float(wd[WD_WOUT + 8 * c + cb + j]);
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1;
            named_bar_sync(2 + buf, DG_THREADS);                        // FULL[buf]: enc slab, J and coordinates of this tile
            // density L0 exactly as forward_chain forms it; the epilogue keeps the ReLU mask, times Woutd[0, :]
            layer<64>([&](float (&d)[32], uint32_t m) { mma_fwd<32, 64>(d, smem_s + S::enc, 4 * buf, smem_s + S::w0d, m); },
                      [&](const float (&d)[32], uint32_t m) {
#pragma unroll
                          for (uint32_t c = 0; c < 8; ++c)
#pragma unroll
                              for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
                                  for (uint32_t j = 0; j < 2; ++j)
                                      s_u[(8 * c + cb + j) * DG_LD + 64 * m + r0 + 8 * h] = d[4 * c + 2 * h + j] > 0.f ? wo[2 * c + j] : 0.f;
                      });
            named_bar_sync(1, 128);                                     // u of every row is in shared memory
            float ge[32];
#pragma unroll
            for (uint32_t k = 0; k < 32; ++k) ge[k] = 0.f;
#pragma unroll 4
            for (uint32_t h = 0; h < 64; ++h) {                         // g_enc = W0d^T u, hidden units in order
                const float uh = s_u[h * DG_LD + t];
                const float4* w = reinterpret_cast<const float4*>(s_w0 + 32 * h);
#pragma unroll
                for (uint32_t q = 0; q < 8; ++q) {
                    const float4 x = w[q];
                    ge[4 * q] = fmaf(uh, x.x, ge[4 * q]); ge[4 * q + 1] = fmaf(uh, x.y, ge[4 * q + 1]);
                    ge[4 * q + 2] = fmaf(uh, x.z, ge[4 * q + 2]); ge[4 * q + 3] = fmaf(uh, x.w, ge[4 * q + 3]);
                }
            }
            const float* jac = reinterpret_cast<const float*>(smem + S::jac + buf * S::jac_bytes);
            float gr[3] = {0.f, 0.f, 0.f};
#pragma unroll
            for (uint32_t k = 0; k < 32; ++k)                           // feature k = 2 level + f, in order
#pragma unroll
                for (uint32_t a = 0; a < 3; ++a) gr[a] = fmaf(jac[(3 * k + a) * DG_LD + t], ge[k], gr[a]);
            if (tile + 2 * gridDim.x < ntiles) named_bar_arrive(4 + buf, DG_THREADS);   // EMPTY[buf]
            const uint32_t row = tile * ROWS + t;
            if (row < n_live) {
                grad_out[3 * (size_t)row] = gr[0]; grad_out[3 * (size_t)row + 1] = gr[1]; grad_out[3 * (size_t)row + 2] = gr[2];
            }
            named_bar_sync(1, 128);                                     // every row has read u before the next tile writes it
        }
    } else {
        const uint32_t tg = t - 128, level = tg & 15, sub = tg >> 4;
        const NgpLevel lv = s_lv[level];
        const __half2* g = reinterpret_cast<const __half2*>(grid) + lv.offset;
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1, row0 = tile * ROWS;
            float* s_coords = reinterpret_cast<float*>(smem + S::coords + buf * 3584);
            if (it >= 2) named_bar_sync(4 + buf, DG_THREADS);           // EMPTY[buf]: the chain of tile it-2 is done with this buffer
            for (uint32_t i = tg; i < ROWS * 7; i += 32 * DG_GW)
                s_coords[i] = (row0 + i / 7 < n_live) ? __ldg(coords + (size_t)row0 * 7 + i) : 0.f;
            named_bar_sync(6, 32 * DG_GW);
            gather_tile_jac(s_coords, lv, g, smem + S::enc, 4 * buf, reinterpret_cast<float*>(smem + S::jac + buf * S::jac_bytes), level, sub);
            fence_proxy_async_smem();                                   // the enc slab is read by the tensor core (async proxy)
            named_bar_arrive(2 + buf, DG_THREADS);                      // FULL[buf]
        }
    }
}

}  // namespace

extern "C" {

int ngp_density_grad(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* grid, const void* levels_dev,
                     const void* w_density, float* grad_out) {
    NGP_REQUIRE(n_max == 0 || (coords != nullptr && grid != nullptr && levels_dev != nullptr && w_density != nullptr),
                "ngp_density_grad: coords, grid, levels and w_density are required");
    NGP_REQUIRE(n_max == 0 || grad_out != nullptr, "ngp_density_grad: grad_out is required");
    if (n_max == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    if (ngp_first_use((const void*)density_grad_kernel))
        NGP_CHECK_CUDA(cudaFuncSetAttribute(density_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmemGrad::total));
    const uint32_t ntiles = (n_max + ROWS - 1) / ROWS;
    const uint32_t grid_dim = min(ntiles, (uint32_t)ngp_num_sms());
    density_grad_kernel<<<grid_dim, DG_THREADS, SmemGrad::total, s>>>(n_max, n_dev, coords, (const __half*)grid, (const NgpLevel*)levels_dev,
                                                                      (const __half*)w_density, grad_out);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
