// R7: the fully-fused MLP as a standalone operator pair (FMLP / FullyFusedMlp_weight boundary,
// OPS/fully_fused_mlp.py:12-145) on Hopper wgmma.
//
// Forward:  persistent CTAs of one warpgroup (128 threads), one 128-row tile at a time.  Weights (<= 30 KB) are staged once per
//   CTA in the canonical K-major GMMA layout; the input tile is written straight into an operand slab; each layer is
//   K/16 wgmma (M=64 per row block, N=64 or 16) into registers; the epilogue (ReLU -> fp16) writes the next layer's operand slab,
//   from which the `output_intermediate` block the reference keeps for backward is copied out row by row.
// Backward: dgrad chain through the same slabs with the weight tiles read MN-major (no transposed copy), and the
//   weight gradients accumulated across all tiles of the CTA in registers (wgrad = dY^T A with both operands read
//   MN-major from the gradient / activation slabs), flushed once with fp32 reductions.  This replaces the reference's
//   kernel_mlp_fused_backward + 5 cuBLAS GEMMs with K = batch (fully_fused_mlp.py:123-143).
// Roofline: tensor (DESIGN.md): 20 480 flop/sample fwd for the two NGP nets, 61 440 fwd+dgrad+wgrad.
#include "mlp_tc.cuh"
#include <cstdlib>

namespace {
using namespace mlp;

constexpr int IN = 32, WIDTH = 64, OUTP = 16;
constexpr int MAX_HM = 3;


struct FwdSmem {
    // slab ping-pong: 2 x 8 groups
    static constexpr uint32_t slab0 = 0, slab1 = 8 * GB;
    static constexpr uint32_t w0 = 16 * GB;                       // 64x32 -> 4 KB
    static constexpr uint32_t wh = w0 + WIDTH * IN * 2;           // n_hm x 8 KB
    __host__ __device__ static constexpr uint32_t wout(uint32_t nhm) { return wh + nhm * WIDTH * WIDTH * 2; }
    __host__ __device__ static constexpr uint32_t total(uint32_t nhm) { return wout(nhm) + OUTP * WIDTH * 2; }
};

__global__ void __launch_bounds__(128)
mlp_fwd_kernel(const __half* __restrict__ W, const __half* __restrict__ X, __half* __restrict__ inter, __half* __restrict__ Y,
               uint32_t nhm, uint32_t n) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t t = threadIdx.x;

    stage_weights(smem + FwdSmem::w0, W, WIDTH, IN, t, 128);
    for (uint32_t j = 0; j < nhm; ++j)
        stage_weights(smem + FwdSmem::wh + j * WIDTH * WIDTH * 2, W + WIDTH * IN + j * WIDTH * WIDTH, WIDTH, WIDTH, t, 128);
    stage_weights(smem + FwdSmem::wout(nhm), W + WIDTH * IN + nhm * WIDTH * WIDTH, OUTP, WIDTH, t, 128);
    const uint32_t smem_s = smem_u32(smem);
    const uint32_t r0 = frag_row(t), cb = (t & 3u) * 4u;

    const uint32_t ntiles = (n + ROWS - 1) / ROWS;
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const uint32_t row = tile * ROWS + t;
        const bool valid = row < n;
        __syncthreads();                                          // the previous tile's last wgmmas have read slab0
        // input row -> slab0 groups 0..3
        {
            const uint4* src = reinterpret_cast<const uint4*>(X + (size_t)row * IN);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                uint4 v = valid ? __ldg(src + g) : make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4*>(smem + FwdSmem::slab0 + g * GB + t * 16) = v;
            }
        }
        operands_ready(0, 128);
        uint32_t cur = FwdSmem::slab0, nxt = FwdSmem::slab1;
        // layer 0
        layer<WIDTH>([&](float (&d)[WIDTH / 2], uint32_t m) { mma_fwd<IN, WIDTH>(d, smem_s + cur, 0, smem_s + FwdSmem::w0, m); },
                     [&](const float (&d)[WIDTH / 2], uint32_t m) { frag_to_slab<WIDTH, true>(d, smem + nxt, 0, m, t); });
        operands_ready(0, 128);
        if (inter && valid) slab_row_to_global(smem + nxt, 0, t, inter + ((size_t)0 * n + row) * WIDTH);
        { uint32_t s = cur; cur = nxt; nxt = s; }
        for (uint32_t j = 0; j < nhm; ++j) {
            const uint32_t w_s = smem_s + FwdSmem::wh + j * WIDTH * WIDTH * 2;
            layer<WIDTH>([&](float (&d)[WIDTH / 2], uint32_t m) { mma_fwd<WIDTH, WIDTH>(d, smem_s + cur, 0, w_s, m); },
                         [&](const float (&d)[WIDTH / 2], uint32_t m) { frag_to_slab<WIDTH, true>(d, smem + nxt, 0, m, t); });
            operands_ready(0, 128);
            if (inter && valid) slab_row_to_global(smem + nxt, 0, t, inter + ((size_t)(j + 1) * n + row) * WIDTH);
            { uint32_t s = cur; cur = nxt; nxt = s; }
        }
        layer<OUTP>([&](float (&d)[OUTP / 2], uint32_t m) { mma_fwd<WIDTH, OUTP>(d, smem_s + cur, 0, smem_s + FwdSmem::wout(nhm), m); },
                    [&](const float (&d)[OUTP / 2], uint32_t m) {
#pragma unroll
                        for (uint32_t h = 0; h < 2; ++h) {
                            const uint32_t r = tile * ROWS + 64 * m + r0 + 8 * h;
                            if (r < n) {
#pragma unroll
                                for (uint32_t c = 0; c < 2; ++c)
                                    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(Y + (size_t)r * OUTP + 8 * c) + cb) =
                                        pack_half2(d[4 * c + 2 * h], d[4 * c + 2 * h + 1]);
                            }
                        }
                    });
    }
}

// ------------------------------------------------------------------------------------------------------
// Backward.  Slab map (groups of 8 features):
//   ACT: [0,4) X | [4+8k, 12+8k) hidden k                       (nh = nhm+1 hidden layers)
//   GRD: [0,2) dY | [2+8j, 10+8j) gradient block j (j=0: last hidden layer ... j=nhm: first)   -- `temps` order
// Weight-gradient accumulators (registers, all tiles of the CTA): Wout as [64 in][16 out], Wh_k and W0 as [64 out][in].
struct BwdLayout {
    uint32_t nhm;
    __host__ __device__ uint32_t act_groups() const { return 4 + 8 * (nhm + 1); }
    __host__ __device__ uint32_t grd_groups() const { return 2 + 8 * (nhm + 1); }
    __host__ __device__ uint32_t act() const { return 0; }
    __host__ __device__ uint32_t grd() const { return act_groups() * GB; }
    // 8 spare groups so that a 64-feature MN-major read starting at the last gradient block stays in bounds
    __host__ __device__ uint32_t w0() const { return grd() + (grd_groups() + 8) * GB; }
    __host__ __device__ uint32_t wh() const { return w0() + WIDTH * IN * 2; }
    __host__ __device__ uint32_t wout() const { return wh() + nhm * WIDTH * WIDTH * 2; }
    __host__ __device__ uint32_t total() const { return wout() + OUTP * WIDTH * 2; }
};

template <uint32_t NHM>
__global__ void __launch_bounds__(128)
mlp_bwd_kernel(const __half* __restrict__ W, const __half* __restrict__ X, const __half* __restrict__ inter,
               const __half* __restrict__ dY, int dy_feature_major, __half* __restrict__ dX, __half* __restrict__ temps,
               float* __restrict__ dW, uint32_t n_out_valid, uint32_t n) {
    // dW == nullptr: dgrad chain only (the link-level mlp_fused_backward_func contract, compat_tcnn.cu); X may then be nullptr.
    // dy_feature_major: dY is (16, n) -- the transposed gradient the reference hands to its backward (fully_fused_mlp.py:117).
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr BwdLayout L{NHM};
    constexpr uint32_t nh = NHM + 1;
    const uint32_t t = threadIdx.x;

    stage_weights(smem + L.w0(), W, WIDTH, IN, t, 128);
    for (uint32_t j = 0; j < NHM; ++j)
        stage_weights(smem + L.wh() + j * WIDTH * WIDTH * 2, W + WIDTH * IN + j * WIDTH * WIDTH, WIDTH, WIDTH, t, 128);
    stage_weights(smem + L.wout(), W + WIDTH * IN + NHM * WIDTH * WIDTH, OUTP, WIDTH, t, 128);
    // spare groups after GRD are read (and ignored) by 64-feature weight-gradient operands: keep them finite
    for (uint32_t i = t; i < 8 * GB / 16; i += 128)
        *reinterpret_cast<uint4*>(smem + L.grd() + L.grd_groups() * GB + i * 16) = make_uint4(0, 0, 0, 0);
    const uint32_t smem_s = smem_u32(smem);
    const uint32_t act_s = smem_s + L.act(), grd_s = smem_s + L.grd();
    uint8_t* act = smem + L.act();
    uint8_t* grd = smem + L.grd();
    const uint32_t r0 = frag_row(t), cb = (t & 3u) * 4u;
    float a_wout[8], a_wh[NHM > 0 ? NHM : 1][32], a_w0[16];   // weight-gradient accumulators

    const uint32_t ntiles = (n + ROWS - 1) / ROWS;
    uint32_t acc = 0;   // 0 on the CTA's first tile: weight-gradient accumulators are overwritten
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, acc = 1) {
        const uint32_t row = tile * ROWS + t;
        const bool valid = row < n;
        const uint4 z = make_uint4(0, 0, 0, 0);
        __syncthreads();                                          // the previous tile's wgmmas have read the slabs
        {
            const uint4* src = reinterpret_cast<const uint4*>(X + (size_t)row * IN);
#pragma unroll
            for (int g = 0; g < 4; ++g) *reinterpret_cast<uint4*>(act + g * GB + t * 16) = (valid && X) ? __ldg(src + g) : z;
            for (uint32_t k = 0; k < nh; ++k) {
                const uint4* hs = reinterpret_cast<const uint4*>(inter + ((size_t)k * n + row) * WIDTH);
#pragma unroll
                for (int g = 0; g < 8; ++g) *reinterpret_cast<uint4*>(act + (4 + 8 * k + g) * GB + t * 16) = valid ? __ldg(hs + g) : z;
            }
            uint4 d0 = z, d1 = z;
            if (valid && !dy_feature_major) {
                const uint4* ds = reinterpret_cast<const uint4*>(dY + (size_t)row * OUTP);
                d0 = __ldg(ds);
                d1 = __ldg(ds + 1);
            } else if (valid) {                       // column c of this row sits at dY[c * n + row]: coalesced across the tile
                __align__(16) __half col[OUTP];
#pragma unroll
                for (int c = 0; c < OUTP; ++c) col[c] = __ldg(dY + (size_t)c * n + row);
                d0 = *reinterpret_cast<const uint4*>(col);
                d1 = *reinterpret_cast<const uint4*>(col + 8);
            }
            *reinterpret_cast<uint4*>(grd + 0 * GB + t * 16) = d0;
            *reinterpret_cast<uint4*>(grd + 1 * GB + t * 16) = d1;
        }
        operands_ready(0, 128);
        // gradient at the last hidden layer, and the output layer's weight gradient [in][out] = h_last^T dY
        if (dW) { wgmma_fence(); mma_wgrad<OUTP>(a_wout, act_s, 4 + 8 * (nh - 1), grd_s, 0, acc); }
        layer<WIDTH>([&](float (&d)[WIDTH / 2], uint32_t m) { mma_dgrad<OUTP, WIDTH>(d, grd_s, 0, smem_s + L.wout(), m); },
                     [&](const float (&d)[WIDTH / 2], uint32_t m) { frag_dgrad_mask<WIDTH>(d, act, 4 + 8 * (nh - 1), grd, 2, m, t); });
        operands_ready(0, 128);
        if (temps && valid) slab_row_to_global(grd, 2, t, temps + ((size_t)0 * n + row) * WIDTH);
        // hidden matmuls, last to first: Wh_{k-1} maps hidden k-1 -> hidden k; its weight gradient [out][in] = g_k^T h_{k-1}
#pragma unroll
        for (uint32_t k = nh - 1; k >= 1; --k) {
            const uint32_t j = nh - 1 - k;            // gradient block holding g_k
            if (dW) { wgmma_fence(); mma_wgrad<WIDTH>(a_wh[k - 1], grd_s, 2 + 8 * j, act_s, 4 + 8 * (k - 1), acc); }
            const uint32_t w_s = smem_s + L.wh() + (k - 1) * WIDTH * WIDTH * 2;
            layer<WIDTH>([&](float (&d)[WIDTH / 2], uint32_t m) { mma_dgrad<WIDTH, WIDTH>(d, grd_s, 2 + 8 * j, w_s, m); },
                         [&](const float (&d)[WIDTH / 2], uint32_t m) { frag_dgrad_mask<WIDTH>(d, act, 4 + 8 * (k - 1), grd, 2 + 8 * (j + 1), m, t); });
            operands_ready(0, 128);
            if (temps && valid) slab_row_to_global(grd, 2 + 8 * (j + 1), t, temps + ((size_t)(j + 1) * n + row) * WIDTH);
        }
        // first layer: dX = g_0 * W0, weight gradient W0 [out][in] = g_0^T X
        if (!dX && !dW) continue;     // dgrad-only call without dL/dinput: nothing left for this tile (uniform over the CTA)
        if (dW) {
            wgmma_fence();
            mma_wgrad<IN>(a_w0, grd_s, 2 + 8 * NHM, act_s, 0, acc);
            wgmma_commit();
        }
        if (dX) {
            layer<IN>([&](float (&d)[IN / 2], uint32_t m) { mma_dgrad<WIDTH, IN>(d, grd_s, 2 + 8 * NHM, smem_s + L.w0(), m); },
                      [&](const float (&d)[IN / 2], uint32_t m) {
#pragma unroll
                          for (uint32_t h = 0; h < 2; ++h) {
                              const uint32_t r = tile * ROWS + 64 * m + r0 + 8 * h;
                              if (r < n) {
#pragma unroll
                                  for (uint32_t c = 0; c < IN / 8; ++c)
                                      *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(dX + (size_t)r * IN + 8 * c) + cb) =
                                          pack_half2(d[4 * c + 2 * h], d[4 * c + 2 * h + 1]);
                              }
                          }
                      });
        }
        wgmma_wait<0>();
    }
    // flush the weight gradients
    if (acc && dW) {
        float* dW0 = dW;
        float* dWh = dW + WIDTH * IN;
        float* dWo = dWh + NHM * WIDTH * WIDTH;
        frag_red_add<OUTP>(a_wout, dWo, 1, WIDTH, WIDTH, n_out_valid, t);
#pragma unroll
        for (uint32_t k = 1; k <= NHM; ++k) frag_red_add<WIDTH>(a_wh[k - 1], dWh + (k - 1) * WIDTH * WIDTH, WIDTH, 1, WIDTH, WIDTH, t);
        frag_red_add<IN>(a_w0, dW0, IN, 1, WIDTH, IN, t);
    }
}

int* g_err_flag = nullptr;
int* err_flag() {
    if (!g_err_flag) {
        if (cudaMalloc(&g_err_flag, sizeof(int)) != cudaSuccess) return nullptr;
        cudaMemset(g_err_flag, 0, sizeof(int));
    }
    return g_err_flag;
}

}  // namespace

int* ngp_err_flag() { return err_flag(); }

extern "C" {


// Debug aid: 1 if any bounded mbarrier wait of a fused kernel timed out since the last call (synchronises the device).
int ngp_debug_timeout_flag(void) {
    int* f = err_flag();
    if (!f) return -1;
    int h = 0;
    if (cudaMemcpy(&h, f, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    if (h) cudaMemset(f, 0, sizeof(int));
    return h;
}

int ngp_mlp_param_count(uint32_t nhm) { return WIDTH * IN + nhm * WIDTH * WIDTH + OUTP * WIDTH; }

int ngp_mlp_fwd(void* stream, const void* weights, const void* input, void* inter, void* output, uint32_t nhm, uint32_t n) {
    NGP_REQUIRE(nhm <= MAX_HM, "ngp_mlp_fwd: at most 3 hidden matmuls (not supported WIDTH/depth)");
    if (n == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t smem = FwdSmem::total(nhm);
    if (ngp_first_use((const void*)mlp_fwd_kernel)) NGP_CHECK_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FwdSmem::total(MAX_HM)));
    const uint32_t ntiles = (n + ROWS - 1) / ROWS;
    const uint32_t grid = min(ntiles, (uint32_t)ngp_num_sms() * 4u);
    mlp_fwd_kernel<<<grid, 128, smem, s>>>((const __half*)weights, (const __half*)input, (__half*)inter, (__half*)output, nhm, n);
    NGP_LAUNCH_CHECK();
    return 0;
}

static int mlp_bwd_launch(void* stream, const void* weights, const void* input, const void* inter, const void* dY, int dy_feature_major,
                          void* dX, void* temps, float* dW, uint32_t nhm, uint32_t n_out_valid, uint32_t n) {
    cudaStream_t s = (cudaStream_t)stream;
    if (dW) NGP_CHECK_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * ngp_mlp_param_count(nhm), s));
    if (n == 0) return 0;
    const BwdLayout L{nhm};
    void (*kernel)(const __half*, const __half*, const __half*, const __half*, int, __half*, __half*, float*, uint32_t, uint32_t) =
        nhm == 0 ? mlp_bwd_kernel<0> : nhm == 1 ? mlp_bwd_kernel<1> : nhm == 2 ? mlp_bwd_kernel<2> : mlp_bwd_kernel<3>;
    if (ngp_first_use((const void*)kernel)) NGP_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total()));
    const uint32_t ntiles = (n + ROWS - 1) / ROWS;
    const uint32_t per_sm = L.total() <= 110 * 1024 ? 2u : 1u;
    const uint32_t grid = min(ntiles, (uint32_t)ngp_num_sms() * per_sm);
    kernel<<<grid, 128, L.total(), s>>>((const __half*)weights, (const __half*)input, (const __half*)inter, (const __half*)dY,
                                        dy_feature_major, (__half*)dX, (__half*)temps, dW, n_out_valid, n);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mlp_bwd(void* stream, const void* weights, const void* input, const void* inter, const void* dY, void* dX, void* temps,
                float* dW, uint32_t nhm, uint32_t n_out_valid, uint32_t n) {
    NGP_REQUIRE(nhm <= MAX_HM, "ngp_mlp_bwd: at most 3 hidden matmuls");
    NGP_REQUIRE(dW != nullptr && inter != nullptr && input != nullptr, "ngp_mlp_bwd: input, inter and dW are required");
    return mlp_bwd_launch(stream, weights, input, inter, dY, 0, dX, temps, dW, nhm, n_out_valid, n);
}

int ngp_mlp_bwd_dgrad(void* stream, const void* weights, const void* inter, const void* dY_feature_major, void* dX, void* temps,
                      uint32_t nhm, uint32_t n) {
    NGP_REQUIRE(nhm <= MAX_HM, "ngp_mlp_bwd_dgrad: at most 3 hidden matmuls");
    NGP_REQUIRE(inter != nullptr && (temps != nullptr || dX != nullptr), "ngp_mlp_bwd_dgrad: inter and one of temps / dX are required");
    return mlp_bwd_launch(stream, weights, nullptr, inter, dY_feature_major, 1, dX, temps, nullptr, nhm, 16, n);
}

}  // extern "C"
