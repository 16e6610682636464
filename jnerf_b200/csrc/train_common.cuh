// What the fused backward (fused_net.cu) and the optimizer sweeps (optimizer.cu) must agree on: the layout of the per-CTA
// weight-gradient slots, how many slots a backward fills, the unit of the fixed-point hash-grid gradient and the Adam+EMA update.
#pragma once
#include "ngp_common.cuh"
#include <algorithm>

// flat weight offsets (halfs) inside the two parameter vectors (OPS/fully_fused_mlp.py:26-40)
constexpr int WD_W0 = 0, WD_WOUT = 64 * 32, WD_N = 64 * 32 + 16 * 64;
constexpr int WR_W0 = 0, WR_W1 = 64 * 32, WR_WOUT = 64 * 32 + 64 * 64, WR_N = 64 * 32 + 64 * 64 + 16 * 64;
constexpr int W_PART = WD_N + WR_N;   // one CTA's weight-gradient sums: [dwd | dwr]

// CTAs of the fused backward over n_max rows, one slot each: a CTA walks pairs of 128-row tiles, at most one CTA per SM
inline uint32_t bwd_ctas(uint32_t n_max) {
    const uint32_t ntiles = (n_max + 127) / 128;
    return std::min((ntiles + 1) / 2, (uint32_t)ngp_num_sms());
}

// Fixed-point hash-grid gradient: feature f of entry e is the signed 64-bit integer fx[2e + f] in units of 2^-32.  The unit is below
// the smallest fp16 spacing (2^-24), so every contribution keeps more precision than an fp16 reduction gives it, and a sum cannot wrap
// while it is within the fp16 range: a contribution is clamped to +-65504 first, and 2^31 units of 1 are 2^31 / 65504 > 32 000 of them.
constexpr float FX_SCALE = 4294967296.0f, FX_INV = 1.0f / 4294967296.0f;

// Every operation is spelled out (no compiler-chosen FMA contraction) so that all kernels that inline this -- the single-GPU
// sweeps, their scalar tails and the data-parallel exchange kernel -- produce bit-identical parameters from identical inputs.
__device__ __forceinline__ float adam_one(float g, float& m, float& v, float& master, const AdamArgs& a) {
    g = __fmul_rn(g, a.grad_scale);
    m = __fmaf_rn(a.b1, m, __fmul_rn(1.f - a.b1, g));
    v = __fmaf_rn(a.b2, v, __fmul_rn(__fmul_rn(1.f - a.b2, g), g));
    const float p = __fsub_rn(master, __fdiv_rn(__fmul_rn(m, a.step_size), __fadd_rn(sqrtf(v), a.eps)));          // jt.nn.Adam.step
    master = __fmul_rn(__fmaf_rn(1.f - a.decay, p, __fmul_rn(__fmul_rn(a.decay, master), a.debias_old)), a.debias_new);   // ema.py:33-36
    return master;
}
