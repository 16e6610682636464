/*
 * ngp_oracle.c -- CPU restatement of the JNeRF Instant-NGP hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  The product (libngp_b200.so) never links, imports or calls it.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/python/jnerf/).  Abbreviations:
 *   HE/  models/position_encoders/hash_encoder/      SH/  models/position_encoders/sh_encoder/
 *   DGS/ models/samplers/density_grid_sampler/       OPS/ ops/code_ops/
 *
 * Pinning status (see DESIGN.md "Oracle"):
 *   - hash fwd/bwd, SH, march, compaction, composite fwd/bwd/inference, occupancy-grid maintenance and
 *     pcg32 are pinned against the reference's own kernel sources executed here (oracle/_ref, host shim)
 *     by tests/test_oracle_vs_ref.py; committed goldens under tests/golden/ were generated from _ref.
 *   - the fully-fused MLP (tiny-cuda-nn, binary only in the reference, sm_75/80/86 SASS) and the
 *     Jittor pieces (Adam, EMA application order, normalize, init) are PARITY UNPINNED: restated from
 *     models/networks/ngp_network.py:59-67 (the nn.Linear fallback defines the math),
 *     OPS/fully_fused_mlp.py:26-40 (weight layout) and optims/{adam,ema,expdecay}.py.
 *
 * Floating-point contraction: the reference only ever runs on the GPU, where nvcc contracts a*b+c into
 * FMA.  `fma_mode` (orc_set_fma_mode) selects the arithmetic for the few contraction-sensitive
 * expressions: 1 = GPU semantics (fmaf), 0 = host-shim semantics (separate multiply and add) so the
 * restatement can be pinned bit-for-bit against oracle/_ref's host build.  Compile with -ffp-contract=off.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

typedef _Float16 half_t;

static int g_fma_mode = 1;
void orc_set_fma_mode(int m) { g_fma_mode = m; }
static inline float mad(float a, float b, float c) { return g_fma_mode ? fmaf(a, b, c) : (float)(a * b) + c; }

static inline float h2f(half_t h) { return (float)h; }
static inline half_t f2h(float f) { return (half_t)f; }

/* ------------------------------------------------------------------------------------------------
 * pcg32  (ops/op_include/pcg32/pcg32.h:53-68 seed/next_uint, :103-112 next_float, :145-166 advance)
 * ---------------------------------------------------------------------------------------------- */
#define PCG32_MULT 0x5851f42d4c957f2dULL
typedef struct { uint64_t state, inc; } orc_pcg32;

static inline uint32_t pcg_next_uint(orc_pcg32* r) {
    uint64_t old = r->state;
    r->state = old * PCG32_MULT + r->inc;
    uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
    uint32_t rot = (uint32_t)(old >> 59u);
    return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
}
static inline float pcg_next_float(orc_pcg32* r) {
    union { uint32_t u; float f; } x;
    x.u = (pcg_next_uint(r) >> 9) | 0x3f800000u;
    return x.f - 1.0f;
}
static inline void pcg_advance(orc_pcg32* r, int64_t delta_) {
    uint64_t cur_mult = PCG32_MULT, cur_plus = r->inc, acc_mult = 1u, acc_plus = 0u;
    uint64_t delta = (uint64_t)delta_;
    while (delta > 0) {
        if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
        cur_plus = (cur_mult + 1) * cur_plus;
        cur_mult *= cur_mult;
        delta /= 2;
    }
    r->state = acc_mult * r->state + acc_plus;
}
void orc_pcg32_seed(uint64_t initstate, uint64_t initseq, uint64_t* state_inc) {
    orc_pcg32 r; r.state = 0; r.inc = (initseq << 1u) | 1u;
    pcg_next_uint(&r); r.state += initstate; pcg_next_uint(&r);
    state_inc[0] = r.state; state_inc[1] = r.inc;
}
void orc_pcg32_advance(uint64_t* state_inc, int64_t delta) {
    orc_pcg32 r = {state_inc[0], state_inc[1]}; pcg_advance(&r, delta); state_inc[0] = r.state;
}
float orc_pcg32_next_float(uint64_t* state_inc) {
    orc_pcg32 r = {state_inc[0], state_inc[1]}; float f = pcg_next_float(&r); state_inc[0] = r.state; return f;
}

/* ------------------------------------------------------------------------------------------------
 * R1: hash-grid level table  (HE/grid_encode.py:17-39)
 * ---------------------------------------------------------------------------------------------- */
double orc_hash_offsets(double aabb_scale, int n_levels, int base_resolution, int log2_hashmap_size, uint32_t* offsets) {
    double pls = exp(log(2048.0 * aabb_scale / base_resolution) / (n_levels - 1));
    uint64_t offset = 0;
    for (int i = 0; i < n_levels; ++i) {
        double scale = pow(2.0, i * log2(pls)) * base_resolution - 1.0;
        uint64_t res = (uint64_t)ceil(scale) + 1;
        uint64_t params = res * res * res;
        params = ((params + 7) / 8) * 8;
        if (params > (1ull << log2_hashmap_size)) params = 1ull << log2_hashmap_size;
        offsets[i] = (uint32_t)offset;
        offset += params;
    }
    offsets[n_levels] = (uint32_t)offset;
    return pls;
}

/* ------------------------------------------------------------------------------------------------
 * R2: hash-grid forward  (HE/op_header/HashEncode.h:68-115 hash/index/fract, :117-203 kernel_grid;
 *     launch + layout HE/grid_encode.py:86-124).  x (n,3) f32 in [0,1]; out (n, 2*L), feature 2*level+f.
 * ---------------------------------------------------------------------------------------------- */
/* cfg.hash_func is pasted into the reference's kernel source as get_index(p0,p1,p2) (HE/hash_encoder.py:13-16); both NGP configs
 * use p0 ^ p1 * 19349663 ^ p2 * 83492791 (ngp_base.py:66).  orc_set_hash_primes selects another member of that XOR-of-products family. */
static uint32_t g_hash_prime[3] = {1u, 19349663u, 83492791u};
static float g_reg_scale = 1.0f;       /* data-parallel shards: ngp_composite_loss_bwd's reg_scale (test infrastructure mirrors the product's knob) */
void orc_set_reg_scale(float s) { g_reg_scale = s; }
void orc_set_hash_primes(uint32_t p0, uint32_t p1, uint32_t p2) { g_hash_prime[0] = p0; g_hash_prime[1] = p1; g_hash_prime[2] = p2; }
static inline uint32_t grid_index(uint32_t hashmap_size, uint32_t res, const uint32_t g[3]) {
    uint32_t stride = 1, index = 0;
    for (uint32_t dim = 0; dim < 3 && stride <= hashmap_size; ++dim) { index += g[dim] * stride; stride *= res; }
    if (hashmap_size < stride) index = g[0] * g_hash_prime[0] ^ g[1] * g_hash_prime[1] ^ g[2] * g_hash_prime[2];
    return (index % hashmap_size) * 2;
}
/* The reference evaluates exp2f on the GPU (MUFU.EX2, <= 2 ulp), libm's exp2f is correctly rounded: the two can
 * differ in the last bits, and the finest levels amplify a 1e-7 relative scale error by the resolution (2048).
 * Tests that compare against a GPU run install the device-computed scales here (NULL = compute with libm). */
static const float* g_level_scales = 0;
void orc_set_level_scales(const float* scales) { g_level_scales = scales; }
static inline void level_setup(uint32_t level, uint32_t base_res, float log2_pls, float* scale, uint32_t* res) {
    *scale = g_level_scales ? g_level_scales[level] : exp2f(level * log2_pls) * base_res - 1.0f;  /* HashEncode.h:149 */
    *res = (uint32_t)ceil(*scale) + 1;                        /* :151 */
}
static inline void pos_fract(float in, float scale, float* pos, uint32_t* g) {
    *pos = mad(in, scale, 0.5f);                              /* HashEncode.h:108 (contracted on GPU) */
    int tmp = (int)floorf(*pos);
    *g = (uint32_t)tmp;
    *pos -= (float)tmp;
}

void orc_hash_fwd_f32(uint32_t n, const float* x, const float* grid, const uint32_t* offsets, uint32_t n_levels,
                      uint32_t base_res, float log2_pls, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i)
        for (uint32_t level = 0; level < n_levels; ++level) {
            const float* g = grid + (size_t)offsets[level] * 2;
            uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
            level_setup(level, base_res, log2_pls, &scale, &res);
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            float r0 = 0, r1 = 0;
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                r0 = mad(w, g[index], r0);                    /* HashEncode.h:199, T = float */
                r1 = mad(w, g[index + 1], r1);
            }
            out[(size_t)i * n_levels * 2 + level * 2] = r0;
            out[(size_t)i * n_levels * 2 + level * 2 + 1] = r1;
        }
}
/* T = __half: every term is rounded to half and accumulated in half (HashEncode.h:199). */
void orc_hash_fwd_f16(uint32_t n, const float* x, const half_t* grid, const uint32_t* offsets, uint32_t n_levels,
                      uint32_t base_res, float log2_pls, half_t* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i)
        for (uint32_t level = 0; level < n_levels; ++level) {
            const half_t* g = grid + (size_t)offsets[level] * 2;
            uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
            level_setup(level, base_res, log2_pls, &scale, &res);
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            half_t r0 = 0, r1 = 0;
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                r0 = f2h(h2f(r0) + h2f(f2h(w * h2f(g[index]))));
                r1 = f2h(h2f(r1) + h2f(f2h(w * h2f(g[index + 1]))));
            }
            out[(size_t)i * n_levels * 2 + level * 2] = r0;
            out[(size_t)i * n_levels * 2 + level * 2 + 1] = r1;
        }
}
/* As above but accumulating in fp32 and rounding once: what an fp32-accumulating kernel should give. */
void orc_hash_fwd_f16_acc32(uint32_t n, const float* x, const half_t* grid, const uint32_t* offsets, uint32_t n_levels,
                            uint32_t base_res, float log2_pls, half_t* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i)
        for (uint32_t level = 0; level < n_levels; ++level) {
            const half_t* g = grid + (size_t)offsets[level] * 2;
            uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
            level_setup(level, base_res, log2_pls, &scale, &res);
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            float r0 = 0, r1 = 0;
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                r0 = mad(w, h2f(g[index]), r0);
                r1 = mad(w, h2f(g[index + 1]), r1);
            }
            out[(size_t)i * n_levels * 2 + level * 2] = f2h(r0);
            out[(size_t)i * n_levels * 2 + level * 2 + 1] = f2h(r1);
        }
}
/* corner indices only: (n, L, 8) entry indices (not *2) -- used for bit-exact index parity */
void orc_hash_indices(uint32_t n, const float* x, const uint32_t* offsets, uint32_t n_levels, uint32_t base_res,
                      float log2_pls, uint32_t* idx_out) {
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t level = 0; level < n_levels; ++level) {
            uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
            level_setup(level, base_res, log2_pls, &scale, &res);
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            for (uint32_t idx = 0; idx < 8; ++idx) {
                uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) pl[d] = pg[d] + ((idx >> d) & 1u);
                idx_out[((size_t)i * n_levels + level) * 8 + idx] = offsets[level] + grid_index(size, res, pl) / 2;
            }
        }
}

/* ------------------------------------------------------------------------------------------------
 * R3: hash-grid backward  (HashEncode.h:299-396 kernel_grid_backward; HE/grid_encode.py:131-190).
 *     grid_grad is zeroed first (grid_encode.py:153); atomics become an in-order sum (level-major,
 *     point index ascending) -- the GPU order is nondeterministic, so parity is tolerance-based.
 * ---------------------------------------------------------------------------------------------- */
void orc_hash_bwd_f32(uint32_t n, const float* x, const float* dy, const uint32_t* offsets, uint32_t n_levels,
                      uint32_t base_res, float log2_pls, float* grid_grad) {
    memset(grid_grad, 0, (size_t)offsets[n_levels] * 2 * sizeof(float));
#pragma omp parallel for schedule(static)
    for (int64_t lv = 0; lv < (int64_t)n_levels; ++lv) {
        uint32_t level = (uint32_t)lv;
        float* g = grid_grad + (size_t)offsets[level] * 2;
        uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
        level_setup(level, base_res, log2_pls, &scale, &res);
        for (uint32_t i = 0; i < n; ++i) {
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            float g0 = dy[(size_t)i * n_levels * 2 + level * 2], g1 = dy[(size_t)i * n_levels * 2 + level * 2 + 1];
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                g[index] += g0 * w;
                g[index + 1] += g1 * w;
            }
        }
    }
}
void orc_hash_bwd_f16(uint32_t n, const float* x, const half_t* dy, const uint32_t* offsets, uint32_t n_levels,
                      uint32_t base_res, float log2_pls, half_t* grid_grad) {
    memset(grid_grad, 0, (size_t)offsets[n_levels] * 2 * sizeof(half_t));
#pragma omp parallel for schedule(static)
    for (int64_t lv = 0; lv < (int64_t)n_levels; ++lv) {
        uint32_t level = (uint32_t)lv;
        half_t* g = grid_grad + (size_t)offsets[level] * 2;
        uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
        level_setup(level, base_res, log2_pls, &scale, &res);
        for (uint32_t i = 0; i < n; ++i) {
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            float g0 = h2f(dy[(size_t)i * n_levels * 2 + level * 2]), g1 = h2f(dy[(size_t)i * n_levels * 2 + level * 2 + 1]);
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                g[index] = f2h(h2f(g[index]) + h2f(f2h(g0 * w)));          /* HashEncode.h:345-346 */
                g[index + 1] = f2h(h2f(g[index + 1]) + h2f(f2h(g1 * w)));
            }
        }
    }
}
/* fp32 accumulation of an fp16 dL/dy: the "ideal" sum the nondeterministic fp16 atomics approximate */
void orc_hash_bwd_f16_acc32(uint32_t n, const float* x, const half_t* dy, const uint32_t* offsets, uint32_t n_levels,
                            uint32_t base_res, float log2_pls, float* grid_grad) {
    memset(grid_grad, 0, (size_t)offsets[n_levels] * 2 * sizeof(float));
#pragma omp parallel for schedule(static)
    for (int64_t lv = 0; lv < (int64_t)n_levels; ++lv) {
        uint32_t level = (uint32_t)lv;
        float* g = grid_grad + (size_t)offsets[level] * 2;
        uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
        level_setup(level, base_res, log2_pls, &scale, &res);
        for (uint32_t i = 0; i < n; ++i) {
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            float g0 = h2f(dy[(size_t)i * n_levels * 2 + level * 2]), g1 = h2f(dy[(size_t)i * n_levels * 2 + level * 2 + 1]);
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                g[index] += g0 * w;
                g[index + 1] += g1 * w;
            }
        }
    }
}
/* The exact scatter of an fp32 dL/dy, for error bounds: w is the fp32 corner weight formed as above, dy * w is exact in double
 * (24 + 24 significant bits), and per feature of every entry it returns g = sum dy * w, a = sum |dy * w| and cnt = the number of
 * nonzero contributions.  g is summed in double in row order: its own error, at most cnt * 2^-53 * a, is far below the fp32 error
 * bounds it is compared with. */
void orc_hash_bwd_f64(uint32_t n, const float* x, const float* dy, const uint32_t* offsets, uint32_t n_levels,
                      uint32_t base_res, float log2_pls, double* grid_grad, double* grid_abs, uint32_t* grid_cnt) {
    const size_t np = (size_t)offsets[n_levels] * 2;
    memset(grid_grad, 0, np * sizeof(double));
    memset(grid_abs, 0, np * sizeof(double));
    memset(grid_cnt, 0, np * sizeof(uint32_t));
#pragma omp parallel for schedule(static)
    for (int64_t lv = 0; lv < (int64_t)n_levels; ++lv) {
        uint32_t level = (uint32_t)lv;
        double* g = grid_grad + (size_t)offsets[level] * 2;
        double* a = grid_abs + (size_t)offsets[level] * 2;
        uint32_t* c = grid_cnt + (size_t)offsets[level] * 2;
        uint32_t size = offsets[level + 1] - offsets[level], res; float scale;
        level_setup(level, base_res, log2_pls, &scale, &res);
        for (uint32_t i = 0; i < n; ++i) {
            float pos[3]; uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pos_fract(x[i * 3 + d], scale, &pos[d], &pg[d]);
            const double g01[2] = {dy[(size_t)i * n_levels * 2 + level * 2], dy[(size_t)i * n_levels * 2 + level * 2 + 1]};
            if (g01[0] == 0.0 && g01[1] == 0.0) continue;
            for (uint32_t idx = 0; idx < 8; ++idx) {
                float w = 1; uint32_t pl[3];
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(size, res, pl);
                for (uint32_t f = 0; f < 2; ++f) {
                    const double v = g01[f] * (double)w;
                    if (v == 0.0) continue;
                    g[index + f] += v;
                    a[index + f] += fabs(v);
                    c[index + f] += 1;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------------
 * R4: spherical harmonics, degree 4  (SH/op_header/SphericalEncode.h:65-95; SH/sh_encoder.py:16)
 * ---------------------------------------------------------------------------------------------- */
static inline void sh4(float dx, float dy, float dz, float* o) {
    float x = dx * 2.f - 1.f, y = dy * 2.f - 1.f, z = dz * 2.f - 1.f;
    if (g_fma_mode) { x = fmaf(dx, 2.f, -1.f); y = fmaf(dy, 2.f, -1.f); z = fmaf(dz, 2.f, -1.f); } /* exact either way */
    float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}
void orc_sh_f32(uint32_t n, const float* dirs, float* out) {
    for (uint32_t i = 0; i < n; ++i) sh4(dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2], out + (size_t)i * 16);
}
void orc_sh_f16(uint32_t n, const float* dirs, half_t* out) {
    for (uint32_t i = 0; i < n; ++i) {
        float o[16]; sh4(dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2], o);
        for (int k = 0; k < 16; ++k) out[(size_t)i * 16 + k] = f2h(o[k]);
    }
}

/* ------------------------------------------------------------------------------------------------
 * R7: bias-free ReLU MLP, fp16 storage.  PARITY UNPINNED (tiny-cuda-nn binary).  Math from
 *     models/networks/ngp_network.py:59-67; flat weight layout from OPS/fully_fused_mlp.py:26-40:
 *     W_flat = [W0 (width x in) | Wh (width x width) * n_hidden_matmuls | Wout (out_pad x width)],
 *     each (out,in) row-major.  inter block k (rows [k*n,(k+1)*n)) = post-ReLU hidden layer k
 *     (fully_fused_mlp.py:133-142).  Accumulation fp32, activations rounded to fp16 per layer.
 * ---------------------------------------------------------------------------------------------- */
void orc_mlp_fwd(uint32_t n, uint32_t in_dim, uint32_t width, uint32_t out_pad, uint32_t n_hidden_matmuls,
                 const half_t* W, const half_t* X, half_t* inter, half_t* Y) {
    const half_t* W0 = W;
    const half_t* Wh = W + (size_t)width * in_dim;
    const half_t* Wo = Wh + (size_t)n_hidden_matmuls * width * width;
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < (int64_t)n; ++s) {
        float a[256], b[256];
        for (uint32_t k = 0; k < in_dim; ++k) a[k] = h2f(X[s * in_dim + k]);
        uint32_t cur = in_dim;
        for (uint32_t l = 0; l <= n_hidden_matmuls; ++l) {
            const half_t* Wl = (l == 0) ? W0 : Wh + (size_t)(l - 1) * width * width;
            for (uint32_t o = 0; o < width; ++o) {
                float acc = 0;
                for (uint32_t k = 0; k < cur; ++k) acc += a[k] * h2f(Wl[o * cur + k]);
                acc = acc > 0 ? acc : 0;
                half_t hv = f2h(acc);
                b[o] = h2f(hv);
                if (inter) inter[((size_t)l * n + s) * width + o] = hv;
            }
            memcpy(a, b, sizeof(float) * width);
            cur = width;
        }
        for (uint32_t o = 0; o < out_pad; ++o) {
            float acc = 0;
            for (uint32_t k = 0; k < width; ++k) acc += a[k] * h2f(Wo[o * width + k]);
            Y[s * out_pad + o] = f2h(acc);
        }
    }
}
/* Backward (OPS/fully_fused_mlp.py:88-145).  dY (n,out_pad) row-major.  temps block j holds the gradient at
 * hidden layer (n_hidden_matmuls - j) -- reverse order, :127-142.  dW (fp32, same flat layout); rows >= n_out_valid
 * of the last layer are zeroed (:136).  dX may be NULL. */
void orc_mlp_bwd(uint32_t n, uint32_t in_dim, uint32_t width, uint32_t out_pad, uint32_t n_hidden_matmuls,
                 uint32_t n_out_valid, const half_t* W, const half_t* X, const half_t* inter, const half_t* dY,
                 half_t* dX, half_t* temps, float* dW) {
    const uint32_t nh = n_hidden_matmuls + 1; /* hidden layers */
    const size_t nW = (size_t)width * in_dim + (size_t)n_hidden_matmuls * width * width + (size_t)out_pad * width;
    const half_t* W0 = W;
    const half_t* Wh = W + (size_t)width * in_dim;
    const half_t* Wo = Wh + (size_t)n_hidden_matmuls * width * width;
    double* acc = (double*)calloc(nW, sizeof(double));
#pragma omp parallel
    {
    double* acc_t = (double*)calloc(nW, sizeof(double));       /* per-thread partial sums, reduced in thread order below */
    float* g = (float*)malloc(sizeof(float) * 2 * width);
#pragma omp for schedule(static)
    for (int64_t ss = 0; ss < (int64_t)n; ++ss) {
        const uint32_t s = (uint32_t)ss;
        float* gc = g; float* gn = g + width;
        /* last hidden layer */
        const half_t* hl = inter + ((size_t)(nh - 1) * n + s) * width;
        for (uint32_t k = 0; k < width; ++k) {
            float a = 0;
            for (uint32_t o = 0; o < out_pad; ++o) a += h2f(dY[(size_t)s * out_pad + o]) * h2f(Wo[o * width + k]);
            gc[k] = h2f(f2h(h2f(hl[k]) > 0 ? a : 0));
        }
        /* wgrad of the output layer */
        double* aWo = acc_t + (size_t)width * in_dim + (size_t)n_hidden_matmuls * width * width;
        for (uint32_t o = 0; o < n_out_valid; ++o)
            for (uint32_t k = 0; k < width; ++k) aWo[o * width + k] += (double)h2f(dY[(size_t)s * out_pad + o]) * h2f(hl[k]);
        if (temps) for (uint32_t k = 0; k < width; ++k) temps[((size_t)0 * n + s) * width + k] = f2h(gc[k]);
        for (int l = (int)nh - 1; l >= 1; --l) { /* hidden matmul l maps hidden l-1 -> hidden l */
            const half_t* Wl = Wh + (size_t)(l - 1) * width * width;
            const half_t* hp = inter + ((size_t)(l - 1) * n + s) * width;
            double* aW = acc_t + (size_t)width * in_dim + (size_t)(l - 1) * width * width;
            for (uint32_t o = 0; o < width; ++o)
                for (uint32_t k = 0; k < width; ++k) aW[o * width + k] += (double)gc[o] * h2f(hp[k]);
            for (uint32_t k = 0; k < width; ++k) {
                float a = 0;
                for (uint32_t o = 0; o < width; ++o) a += gc[o] * h2f(Wl[o * width + k]);
                gn[k] = h2f(f2h(h2f(hp[k]) > 0 ? a : 0));
            }
            float* t = gc; gc = gn; gn = t;
            if (temps) for (uint32_t k = 0; k < width; ++k) temps[((size_t)(nh - l) * n + s) * width + k] = f2h(gc[k]);
        }
        for (uint32_t o = 0; o < width; ++o)
            for (uint32_t k = 0; k < in_dim; ++k) acc_t[o * in_dim + k] += (double)gc[o] * h2f(X[(size_t)s * in_dim + k]);
        if (dX)
            for (uint32_t k = 0; k < in_dim; ++k) {
                float a = 0;
                for (uint32_t o = 0; o < width; ++o) a += gc[o] * h2f(W0[o * in_dim + k]);
                dX[(size_t)s * in_dim + k] = f2h(a);
            }
    }
#pragma omp critical
    for (size_t i = 0; i < nW; ++i) acc[i] += acc_t[i];
    free(acc_t); free(g);
    }
    for (size_t i = 0; i < nW; ++i) dW[i] = (float)acc[i];
    free(acc);
}

/* ------------------------------------------------------------------------------------------------
 * NGP network forward (models/networks/ngp_network.py:77-89): out (n,4) = [rgb(3), density h[:,0]].
 * density net 32->64->16, rgb net [h16 | sh16]->64->64->16(3 valid).  Also returns enc/h if non-NULL.
 * ---------------------------------------------------------------------------------------------- */
void orc_network_fwd(uint32_t n, const float* pos, const float* dir, const half_t* grid, const uint32_t* offsets,
                     uint32_t n_levels, uint32_t base_res, float log2_pls, const half_t* Wd, const half_t* Wr,
                     int acc32, half_t* out4, half_t* enc_out, half_t* h_out) {
    half_t* enc = (half_t*)malloc((size_t)n * 32 * sizeof(half_t));
    half_t* h = (half_t*)malloc((size_t)n * 16 * sizeof(half_t));
    half_t* rin = (half_t*)malloc((size_t)n * 32 * sizeof(half_t));
    half_t* r = (half_t*)malloc((size_t)n * 16 * sizeof(half_t));
    if (acc32) orc_hash_fwd_f16_acc32(n, pos, grid, offsets, n_levels, base_res, log2_pls, enc);
    else orc_hash_fwd_f16(n, pos, grid, offsets, n_levels, base_res, log2_pls, enc);
    orc_mlp_fwd(n, 32, 64, 16, 0, Wd, enc, NULL, h);
    for (uint32_t i = 0; i < n; ++i) {
        float o[16]; sh4(dir[i * 3], dir[i * 3 + 1], dir[i * 3 + 2], o);
        for (int k = 0; k < 16; ++k) { rin[(size_t)i * 32 + k] = h[(size_t)i * 16 + k]; rin[(size_t)i * 32 + 16 + k] = f2h(o[k]); }
    }
    orc_mlp_fwd(n, 32, 64, 16, 1, Wr, rin, NULL, r);
    for (uint32_t i = 0; i < n; ++i) {
        out4[(size_t)i * 4 + 0] = r[(size_t)i * 16 + 0]; out4[(size_t)i * 4 + 1] = r[(size_t)i * 16 + 1];
        out4[(size_t)i * 4 + 2] = r[(size_t)i * 16 + 2]; out4[(size_t)i * 4 + 3] = h[(size_t)i * 16];
    }
    if (enc_out) memcpy(enc_out, enc, (size_t)n * 32 * sizeof(half_t));
    if (h_out) memcpy(h_out, h, (size_t)n * 16 * sizeof(half_t));
    free(enc); free(h); free(rin); free(r);
}

/* ------------------------------------------------------------------------------------------------
 * R6: ray march  (DGS/op_header/ray_sampler.h:4-114 + helpers in ray_sampler_header.h:
 *     BoundingBox::ray_intersect :408-465, contains :472-477, mip_from_pos/dt :60-77, morton :642-657,
 *     distance/advance_to_next_voxel :728-753, cascaded_grid_idx_at/occupied :755-776, warp_* :790-843;
 *     calc_dt generated at DGS/density_grid_sampler.py:107-115).
 *     Output order: the reference claims output ranges with atomicAdd (nondeterministic); here and in the
 *     CUDA product the base of ray i is the exclusive prefix sum of numsteps in ray order.
 * ---------------------------------------------------------------------------------------------- */
#define NERF_GRIDSIZE 128u
#define NERF_STEPS 1024u
static const float SQRT3_ = 1.73205080757f;
typedef struct { uint32_t cascades; int const_dt; float min_cone, max_cone; } march_cfg;
static march_cfg make_cfg(uint32_t cascades, int const_dt) {
    march_cfg c; c.cascades = cascades; c.const_dt = const_dt;
    c.min_cone = SQRT3_ / NERF_STEPS;
    c.max_cone = (SQRT3_ / NERF_STEPS) * (1 << (cascades - 1)) * NERF_STEPS / NERF_GRIDSIZE;
    return c;
}
static inline float calc_dt(const march_cfg* c, float t, float cone) {
    if (c->const_dt) return (float)(c->min_cone * 0.5); /* MIN_CONE_STEPSIZE() * 0.5 (double literal) */
    float v = t * cone;
    return v < c->min_cone ? c->min_cone : (c->max_cone < v ? c->max_cone : v);
}
static inline uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu; v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u; v = (v * 0x00000005u) & 0x49249249u; return v;
}
static inline uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) { return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2); }
static inline uint32_t morton3D_invert(uint32_t x) {
    x = x & 0x49249249; x = (x | (x >> 2)) & 0xc30c30c3; x = (x | (x >> 4)) & 0x0f00f00f;
    x = (x | (x >> 8)) & 0xff0000ff; x = (x | (x >> 16)) & 0x0000ffff; return x;
}
uint32_t orc_morton3D(uint32_t x, uint32_t y, uint32_t z) { return morton3D(x, y, z); }
uint32_t orc_morton3D_invert(uint32_t x) { return morton3D_invert(x); }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }
static inline int mip_from_pos(const march_cfg* c, const float p[3]) {
    int e; float m = fmaxf(fmaxf(fabsf(p[0] - 0.5f), fabsf(p[1] - 0.5f)), fabsf(p[2] - 0.5f));
    frexpf(m, &e);
    return imin((int)c->cascades - 1, imax(0, e + 1));
}
static inline int mip_from_dt(const march_cfg* c, float dt, const float p[3]) {
    int mip = mip_from_pos(c, p);
    dt *= 2 * NERF_GRIDSIZE;
    if (dt < 1.f) return mip;
    int e; frexpf(dt, &e);
    return imin((int)c->cascades - 1, imax(e, mip));
}
static inline uint32_t cascaded_grid_idx_at(const float p[3], uint32_t mip) {
    float s = scalbnf(1.0f, -(int)mip);
    int ix[3];
    for (int d = 0; d < 3; ++d) {
        float q = p[d] - 0.5f; q *= s; q += 0.5f;
        int i = (int)(q * NERF_GRIDSIZE);
        ix[d] = i < 0 ? 0 : (i > (int)NERF_GRIDSIZE - 1 ? (int)NERF_GRIDSIZE - 1 : i);
    }
    return morton3D(ix[0], ix[1], ix[2]);
}
static inline int occupied_at(const float p[3], const uint8_t* bits, uint32_t mip) {
    uint32_t idx = cascaded_grid_idx_at(p, mip);
    return bits[idx / 8 + (NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE) * mip / 8] & (1 << (idx % 8));
}
static inline float sgn(float x) { return copysignf(1.0f, x); }
static inline float dist_next_voxel(const float p_[3], const float d[3], const float id[3], uint32_t res) {
    float p[3] = {res * p_[0], res * p_[1], res * p_[2]};
    float tx = (floorf(p[0] + 0.5f + 0.5f * sgn(d[0])) - p[0]) * id[0];
    float ty = (floorf(p[1] + 0.5f + 0.5f * sgn(d[1])) - p[1]) * id[1];
    float tz = (floorf(p[2] + 0.5f + 0.5f * sgn(d[2])) - p[2]) * id[2];
    float t = fminf(fminf(tx, ty), tz);
    return fmaxf(t / res, 0.0f);
}
static inline float advance_next_voxel(const march_cfg* c, float t, float cone, const float p[3], const float d[3],
                                       const float id[3], uint32_t res) {
    float t_target = t + dist_next_voxel(p, d, id, res);
    do { t += calc_dt(c, t, cone); } while (t < t_target);
    return t;
}
static inline int aabb_contains(float lo, float hi, const float p[3]) {
    return p[0] >= lo && p[0] <= hi && p[1] >= lo && p[1] <= hi && p[2] >= lo && p[2] <= hi;
}
static void ray_intersect(float lo, float hi, const float o[3], const float d[3], float* tmin_, float* tmax_) {
    float tmin = (lo - o[0]) / d[0], tmax = (hi - o[0]) / d[0], t;
    if (tmin > tmax) { t = tmin; tmin = tmax; tmax = t; }
    float tymin = (lo - o[1]) / d[1], tymax = (hi - o[1]) / d[1];
    if (tymin > tymax) { t = tymin; tymin = tymax; tymax = t; }
    if (tmin > tymax || tymin > tmax) { *tmin_ = FLT_MAX; *tmax_ = FLT_MAX; return; }
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    float tzmin = (lo - o[2]) / d[2], tzmax = (hi - o[2]) / d[2];
    if (tzmin > tzmax) { t = tzmin; tzmin = tzmax; tzmax = t; }
    if (tmin > tzmax || tzmin > tmax) { *tmin_ = FLT_MAX; *tmax_ = FLT_MAX; return; }
    if (tzmin > tmin) tmin = tzmin;
    if (tzmax < tmax) tmax = tzmax;
    *tmin_ = tmin; *tmax_ = tmax;
}
static inline float warp_dt(const march_cfg* c, float dt) {
    float max_stepsize = c->min_cone * (1 << (c->cascades - 1));
    return (dt - c->min_cone) / (max_stepsize - c->min_cone);
}
static inline float unwarp_dt(const march_cfg* c, float dt) {
    float max_stepsize = c->min_cone * (1 << (c->cascades - 1));
    return mad(dt, max_stepsize - c->min_cone, c->min_cone);
}

/* counters[0] = rays with base in range (ray_counter), counters[1] = total numsteps (incl. overflowing rays).
 * numsteps (R,2) = {count, base}; ray_indices (R): sequential id or 0xFFFFFFFF for empty rays; coords (S,7). */
void orc_march(uint32_t n_rays, float aabb_lo, float aabb_hi, uint32_t max_samples, const float* rays_o,
               const float* rays_d, const uint8_t* bitfield, float cone_angle, float near_distance,
               uint32_t cascades, int const_dt, uint64_t rng_state, uint64_t rng_inc, uint32_t* counters,
               uint32_t* ray_indices, uint32_t* numsteps, float* coords) {
    march_cfg c = make_cfg(cascades, const_dt);
    for (uint32_t i = 0; i < n_rays; ++i) {
        orc_pcg32 rng = {rng_state, rng_inc};
        pcg_advance(&rng, (int64_t)(uint32_t)(i * 8u));         /* ray_sampler.h:30 */
        const float* o = rays_o + 3 * i; const float* d = rays_d + 3 * i;
        float tmin, tmax; ray_intersect(aabb_lo, aabb_hi, o, d, &tmin, &tmax);
        float cone = cone_angle;                                 /* calc_cone_angle returns the constant */
        tmin = fmaxf(tmin, near_distance);
        float startt = tmin;
        startt = mad(calc_dt(&c, startt, cone), pcg_next_float(&rng), startt); /* :48 */
        float id[3] = {1.0f / d[0], 1.0f / d[1], 1.0f / d[2]};
        uint32_t j = 0; float t = startt; float p[3];
        for (;;) {
            p[0] = mad(t, d[0], o[0]); p[1] = mad(t, d[1], o[1]); p[2] = mad(t, d[2], o[2]);
            if (!(aabb_contains(aabb_lo, aabb_hi, p) && j < NERF_STEPS)) break;
            float dt = calc_dt(&c, t, cone);
            uint32_t mip = (uint32_t)mip_from_dt(&c, dt, p);
            if (occupied_at(p, bitfield, mip)) { ++j; t += dt; }
            else t = advance_next_voxel(&c, t, cone, p, d, id, NERF_GRIDSIZE >> mip);
        }
        uint32_t n = j, base = counters[1];
        counters[1] += n;
        if (base + n > max_samples) { numsteps[2 * i] = 0; numsteps[2 * i + 1] = base; continue; }
        uint32_t ray_idx = counters[0]++;
        ray_indices[i] = ray_idx;
        numsteps[2 * i] = n; numsteps[2 * i + 1] = base;
        if (n == 0) { ray_indices[i] = 0xFFFFFFFFu; continue; }
        float wd[3] = {(d[0] + 1.0f) * 0.5f, (d[1] + 1.0f) * 0.5f, (d[2] + 1.0f) * 0.5f};
        float diag = aabb_hi - aabb_lo;
        t = startt; j = 0;
        float* out = coords + (size_t)base * 7;
        for (;;) {
            p[0] = mad(t, d[0], o[0]); p[1] = mad(t, d[1], o[1]); p[2] = mad(t, d[2], o[2]);
            if (!(aabb_contains(aabb_lo, aabb_hi, p) && j < n)) break;
            float dt = calc_dt(&c, t, cone);
            uint32_t mip = (uint32_t)mip_from_dt(&c, dt, p);
            if (occupied_at(p, bitfield, mip)) {
                float* q = out + (size_t)j * 7;
                q[0] = (p[0] - aabb_lo) / diag; q[1] = (p[1] - aabb_lo) / diag; q[2] = (p[2] - aabb_lo) / diag;
                q[3] = warp_dt(&c, dt);
                q[4] = wd[0]; q[5] = wd[1]; q[6] = wd[2];
                ++j; t += dt;
            } else t = advance_next_voxel(&c, t, cone, p, d, id, NERF_GRIDSIZE >> mip);
        }
    }
}

/* R5: compaction (DGS/op_header/compacted_coord.h:4-76).  The transmittance early-out is commented out in the
 * reference (:40-43), so the network output does not influence the result: per-ray copy + truncation. */
void orc_compact(uint32_t n_rays, uint32_t max_compacted, const float* coords_in, const uint32_t* numsteps_in,
                 float* coords_out, uint32_t* numsteps_out, uint32_t* counters /* [0]=numsteps, [1]=rays */) {
    for (uint32_t i = 0; i < n_rays; ++i) {
        uint32_t n = numsteps_in[2 * i], base = numsteps_in[2 * i + 1];
        uint32_t cbase = counters[0]; counters[0] += n;
        uint32_t lim = max_compacted - (max_compacted < cbase ? max_compacted : cbase);
        uint32_t cn = lim < n ? lim : n;
        numsteps_out[2 * i] = cn; numsteps_out[2 * i + 1] = cbase;
        if (cn == 0) continue;
        counters[1]++;
        memcpy(coords_out + (size_t)cbase * 7, coords_in + (size_t)base * 7, (size_t)cn * 7 * sizeof(float));
    }
}

/* ------------------------------------------------------------------------------------------------
 * R8/R9: volume-render composite (DGS/op_header/calc_rgb.h:10-74 fwd, :76-148 bwd, :151-212 inference;
 *        activations ray_sampler_header.h:900-942, derivatives :1018-1058).  net (N,4) = {r,g,b,sigma_raw}.
 * ---------------------------------------------------------------------------------------------- */
static inline float logistic(float x) { return 1.0f / (1.0f + expf(-x)); }
#define NET(k) (is_half ? h2f(((const half_t*)net)[k]) : ((const float*)net)[k])

void orc_composite_fwd(uint32_t n_rays, const void* net, int is_half, const float* coords, const uint32_t* numsteps_in,
                       const uint32_t* numsteps_compacted, const float* bg, uint32_t cascades, float* rgb_out) {
    march_cfg c = make_cfg(cascades, 1);
    for (uint32_t i = 0; i < n_rays; ++i) {
        uint32_t n = numsteps_compacted[2 * i], base = numsteps_compacted[2 * i + 1];
        const float* b = bg + 3 * i;
        if (n == 0) { rgb_out[3 * i] = b[0]; rgb_out[3 * i + 1] = b[1]; rgb_out[3 * i + 2] = b[2]; continue; }
        float T = 1.f, r[3] = {0, 0, 0};
        uint32_t j = 0;
        for (; j < n; ++j) {
            size_t k = (size_t)(base + j) * 4;
            float rgb[3] = {logistic(NET(k)), logistic(NET(k + 1)), logistic(NET(k + 2))};
            float dt = unwarp_dt(&c, coords[(size_t)(base + j) * 7 + 3]);
            float density = expf(NET(k + 3));
            float alpha = 1.f - expf(-density * dt);
            float w = alpha * T;
            r[0] = mad(w, rgb[0], r[0]); r[1] = mad(w, rgb[1], r[1]); r[2] = mad(w, rgb[2], r[2]);
            T *= (1.f - alpha);
        }
        if (j == numsteps_in[2 * i]) { r[0] = mad(T, b[0], r[0]); r[1] = mad(T, b[1], r[1]); r[2] = mad(T, b[2], r[2]); }
        rgb_out[3 * i] = r[0]; rgb_out[3 * i + 1] = r[1]; rgb_out[3 * i + 2] = r[2];
    }
}
void orc_composite_infer(uint32_t n_rays, const void* net, int is_half, const float* coords, const uint32_t* numsteps,
                         uint32_t cascades, float* rgb_out, float* alpha_out) {
    march_cfg c = make_cfg(cascades, 1);
    for (uint32_t i = 0; i < n_rays; ++i) {
        uint32_t n = numsteps[2 * i], base = numsteps[2 * i + 1];
        if (n == 0) { rgb_out[3 * i] = rgb_out[3 * i + 1] = rgb_out[3 * i + 2] = 0; alpha_out[i] = 0; continue; }
        float T = 1.f, r[3] = {0, 0, 0};
        for (uint32_t j = 0; j < n; ++j) {
            size_t k = (size_t)(base + j) * 4;
            float rgb[3] = {logistic(NET(k)), logistic(NET(k + 1)), logistic(NET(k + 2))};
            float dt = unwarp_dt(&c, coords[(size_t)(base + j) * 7 + 3]);
            float alpha = 1.f - expf(-expf(NET(k + 3)) * dt);
            float w = alpha * T;
            r[0] = mad(w, rgb[0], r[0]); r[1] = mad(w, rgb[1], r[1]); r[2] = mad(w, rgb[2], r[2]);
            T *= (1.f - alpha);
        }
        rgb_out[3 * i] = r[0]; rgb_out[3 * i + 1] = r[1]; rgb_out[3 * i + 2] = r[2];
        alpha_out[i] = 1 - T;
    }
}
/* dL/dnet (n_elements,4), zero-filled first (DGS/calc_rgb.py:93). out type = net type. */
void orc_composite_bwd(uint32_t n_rays, uint32_t n_elements, const void* net, int is_half, const float* coords,
                       const uint32_t* numsteps_compacted, const float* loss_grad, const float* rgb_ray,
                       float density_grid_mean, uint32_t cascades, void* dnet) {
    march_cfg c = make_cfg(cascades, 1);
    memset(dnet, 0, (size_t)n_elements * 4 * (is_half ? 2 : 4));
    float loss_scale = 128; loss_scale /= n_rays;
    const float l1 = (density_grid_mean < 0.01f ? 1e-4f : 0.0f) * g_reg_scale;
    for (uint32_t i = 0; i < n_rays; ++i) {
        uint32_t n = numsteps_compacted[2 * i], base = numsteps_compacted[2 * i + 1];
        const float* lg = loss_grad + 3 * i; const float* rr = rgb_ray + 3 * i;
        float T = 1.f, r2[3] = {0, 0, 0};
        for (uint32_t j = 0; j < n; ++j) {
            size_t k = (size_t)(base + j) * 4;
            float o[4] = {NET(k), NET(k + 1), NET(k + 2), NET(k + 3)};
            float rgb[3] = {logistic(o[0]), logistic(o[1]), logistic(o[2])};
            float dt = unwarp_dt(&c, coords[(size_t)(base + j) * 7 + 3]);
            float density = expf(o[3]);
            float alpha = 1.f - expf(-density * dt);
            float w = alpha * T;
            for (int q = 0; q < 3; ++q) r2[q] = mad(w, rgb[q], r2[q]);
            T *= (1.f - alpha);
            float suffix[3] = {rr[0] - r2[0], rr[1] - r2[1], rr[2] - r2[2]};
            float dl[4];
            for (int q = 0; q < 3; ++q) {
                float dr = rgb[q] * (1 - rgb[q]);
                dl[q] = loss_scale * ((w * lg[q]) * dr + fmaxf(0.0f, 0.0f * o[q]));
            }
            float cl = o[3] < -15.0f ? -15.0f : (o[3] > 15.0f ? 15.0f : o[3]);
            float dd = expf(cl);
            /* Eigen's fixed-size redux associates a 3-term dot as x0 + (x1 + x2) */
            float dot = lg[0] * (T * rgb[0] - suffix[0]) + (lg[1] * (T * rgb[1] - suffix[1]) + lg[2] * (T * rgb[2] - suffix[2]));
            float dmlp = dd * (dt * dot);
            dl[3] = loss_scale * dmlp + (o[3] < 0 ? -l1 : 0.0f);
            for (int q = 0; q < 4; ++q) {
                if (is_half) ((half_t*)dnet)[k + q] = f2h(dl[q]); else ((float*)dnet)[k + q] = dl[q];
            }
        }
    }
}
/* The composite in float64 with a per-entry error bound for an fp32 evaluation of it (the bound is derived in
 * tests/test_gpu_composite_reference.py).  Every value below is an (exact value, absolute error bound) pair; the rules:
 *   ev_mul / ev_add: a rounded fp32 operation on inputs with errors ea, eb: |a| eb + |b| ea + ea eb, plus u (|v| + e) for the
 *     rounding and 2^-150 for a result in the subnormal range (u = 2^-24);
 *   __expf(x): relative (2 + floor(1.173 |x|)) 2^-23, plus 2^-126 for a flushed subnormal result;
 *   logistic_sfu: __expf, one rounded add, __fdividef (2 ulp = 4u, and 0 for a denominator beyond 2^126, so 2^-126 absolute);
 *   products of m transmittance factors and sums of m non-negative fmaf terms: gamma_m = m u / (1 - m u) of the magnitude, any
 *     association (a sum of m terms in any binary tree rounds at most m times on the way from a term to the result).
 * dt is the kernel's own fp32 value (nerf_unwarp_dt is one fmaf); net rows, bg, lg, rr, loss_scale and l1 are exact inputs.
 * numsteps_in == NULL: inference (no background).  lg == NULL: forward only. */
typedef struct { double v, e; } ev;
#define EV_U 0x1p-24
#define EV_TINY 0x1p-150
static inline ev ev_exact(double v) { ev r = {v, 0.0}; return r; }
static inline ev ev_round(double v, double e) { ev r = {v, e + EV_U * (fabs(v) + e) + EV_TINY}; return r; }
static inline ev ev_mul(ev a, ev b) { return ev_round(a.v * b.v, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e); }
static inline ev ev_add(ev a, ev b) { return ev_round(a.v + b.v, a.e + b.e); }
static inline double expf_rel(double x) { return (2.0 + floor(1.173 * fabs(x))) * 0x1p-23; }
static inline double gamma_m(double m) { return m * EV_U / (1.0 - m * EV_U); }

void orc_composite_f64(uint32_t n_rays, const void* net, int is_half, const float* coords, const uint32_t* numsteps_in,
                       const uint32_t* numsteps_c, const float* bg, uint32_t cascades, float loss_scale, float l1,
                       const float* lg, const float* rr, double* rgb, double* rgb_err, double* T_final, double* T_err,
                       double* alpha, double* alpha_err, double* dnet, double* dnet_err) {
    march_cfg c = make_cfg(cascades, 1);
    const float max_step = c.min_cone * (float)(1u << (cascades - 1)), span = max_step - c.min_cone;
    for (uint32_t i = 0; i < n_rays; ++i) {
        const uint32_t n = numsteps_c[2 * i], base = numsteps_c[2 * i + 1];
        const int full = numsteps_in != NULL && n == numsteps_in[2 * i];
        double T = 1, Tu = 1, Tl = 1;                    /* exact transmittance, and with every factor at its upper / lower bound */
        double P[3] = {0, 0, 0}, D[3] = {0, 0, 0}, M[3] = {0, 0, 0};   /* sum w c, its propagated error, sum of magnitudes */
        for (uint32_t j = 0; j < n; ++j) {
            const size_t k = (size_t)(base + j) * 4;
            const double o[4] = {NET(k), NET(k + 1), NET(k + 2), NET(k + 3)};
            const double dt = fmaf(coords[(size_t)(base + j) * 7 + 3], span, c.min_cone);
            ev col[3];
            for (int q = 0; q < 3; ++q) {
                const double E = exp(-o[q]), cq = 1.0 / (1.0 + E), om = isinf(E) ? 1.0 : E / (1.0 + E);   /* om = 1 - c */
                const double rel = (1 + 4 * EV_U) / ((1 - om * expf_rel(o[q])) * (1 - EV_U)) - 1;
                col[q].v = cq; col[q].e = cq * rel + 0x1p-126;
            }
            /* alpha = 1 - exp(-sigma dt): bracket the kernel's exp(fl(-fl(__expf(o_w)) dt)) */
            const double sig = exp(o[3]), es = expf_rel(o[3]);
            const double z = -sig * dt, E2 = exp(z), a = -expm1(z), f = E2;
            const double zlo = -(sig * (1 + es) + 0x1p-126) * dt * (1 + EV_U), zhi = -fmax(sig * (1 - es) - 0x1p-126, 0.0) * dt * (1 - EV_U);
            const double ez = isinf(zlo) ? 0.0 : expf_rel(zlo);
            const double E2hi = exp(zhi) * (1 + ez) + 0x1p-126, E2lo = fmax(exp(zlo) * (1 - ez) - 0x1p-126, 0.0);
            double A = fmax(E2hi - E2, E2 - E2lo);
            A += EV_U * (a + A);                                             /* alpha = fl(1 - E2) */
            const double Phi = A + EV_U * (f + A);                            /* the factor fl(1 - alpha) */
            const double g_b = gamma_m(j), g_a = gamma_m(j + 1);
            const ev Tb = {T, fmax(Tu - T, T - Tl) + g_b * Tu + j * EV_TINY};
            const ev w = ev_mul((ev){a, A}, Tb);
            T *= f; Tu *= f + Phi; Tl *= fmax(f - Phi, 0.0);
            const ev Ta = {T, fmax(Tu - T, T - Tl) + g_a * Tu + (j + 1) * EV_TINY};
            for (int q = 0; q < 3; ++q) {                                    /* fmaf: the product w c is not rounded on its own */
                const double t = w.v * col[q].v, et = fabs(w.v) * col[q].e + fabs(col[q].v) * w.e + w.e * col[q].e;
                P[q] += t; D[q] += et; M[q] += fabs(t) + et;
            }
            if (lg == NULL) continue;
            ev dl[4], tq[3];
            for (int q = 0; q < 3; ++q) {
                const ev run = {P[q], D[q] + gamma_m(j + 1) * M[q] + (j + 1) * EV_TINY};
                const ev suffix = ev_add(ev_exact(rr[3 * i + q]), (ev){-run.v, run.e});
                const ev tc = ev_mul(Ta, col[q]);
                tq[q] = ev_add(tc, (ev){-suffix.v, suffix.e});
                const ev om = ev_add(ev_exact(1.0), (ev){-col[q].v, col[q].e});
                const ev g = ev_mul(col[q], om);
                dl[q] = ev_mul(ev_exact(loss_scale), ev_mul(ev_mul(w, ev_exact(lg[3 * i + q])), g));
            }
            /* Eigen's fixed-size redux: x0 + (x1 + x2) */
            const ev dot = ev_add(ev_mul(ev_exact(lg[3 * i]), tq[0]),
                         ev_add(ev_mul(ev_exact(lg[3 * i + 1]), tq[1]), ev_mul(ev_exact(lg[3 * i + 2]), tq[2])));
            const float cl = o[3] < -15.0 ? -15.0f : (o[3] > 15.0 ? 15.0f : (float)o[3]);
            const double dd = exp((double)cl);
            dl[3] = ev_mul(ev_exact(loss_scale), ev_mul((ev){dd, dd * expf_rel(cl)}, ev_mul(ev_exact(dt), dot)));
            if (o[3] < 0) dl[3] = ev_add(dl[3], ev_exact(-(double)l1));
            for (int q = 0; q < 4; ++q) { dnet[k + q] = dl[q].v; dnet_err[k + q] = dl[q].e; }
        }
        const double gn = gamma_m(n);
        const ev Tn = {T, n ? fmax(Tu - T, T - Tl) + gn * Tu + n * EV_TINY : 0.0};
        T_final[i] = Tn.v; T_err[i] = Tn.e;
        alpha[i] = n ? 1 - T : 0; alpha_err[i] = n ? Tn.e + EV_U * (1 - T + Tn.e) : 0;
        for (int q = 0; q < 3; ++q) {
            double v = P[q], e = D[q] + gn * M[q] + n * EV_TINY;
            if (numsteps_in != NULL && n == 0) { v = bg[3 * i + q]; e = 0; }
            else if (full) {                                                 /* fmaf(T, bg, r): one more rounding */
                const double b = bg[3 * i + q];
                v = P[q] + T * b;
                e = D[q] + Tn.e * b + gamma_m(n + 1) * (M[q] + (T + Tn.e) * b) + (n + 1) * EV_TINY;
            }
            rgb[3 * i + q] = v; rgb_err[3 * i + q] = e;
        }
    }
}

/* Huber loss gradient (models/losses/huber_loss.py:11-14), unreduced loss summed by Jittor's backward */
void orc_huber_grad(uint32_t n, const float* x, const float* target, float delta, float* grad, float* loss) {
    for (uint32_t i = 0; i < n; ++i) {
        float diff = x[i] - target[i], rel = fabsf(diff);
        if (loss) loss[i] = rel > delta ? rel - 0.5f * delta : 0.5f / delta * rel * rel;
        grad[i] = rel > delta ? (diff > 0 ? 1.0f : -1.0f) : diff / delta;
    }
}

/* ------------------------------------------------------------------------------------------------
 * R10: occupancy-grid maintenance (DGS/density_grid_sampler.py:204-264 and the five small headers)
 * ---------------------------------------------------------------------------------------------- */
/* mark_untrained_density_grid.h:3-48.  xforms (n_img, 3x4 column-major = 12 f32), focal (n_img,2) */
void orc_mark_untrained(uint32_t n_elements, float* grid, uint32_t n_images, const float* focal, const float* xforms,
                        int res_x, int res_y) {
    const uint32_t G3 = NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE;
#pragma omp parallel for schedule(static)
    for (int64_t ii = 0; ii < (int64_t)n_elements; ++ii) {
        uint32_t i = (uint32_t)ii, level = i / G3, pos_idx = i % G3;
        uint32_t x = morton3D_invert(pos_idx >> 0), y = morton3D_invert(pos_idx >> 1), z = morton3D_invert(pos_idx >> 2);
        float half_resx = res_x * 0.5f, half_resy = res_y * 0.5f;
        float sc = scalbnf(1.0f, (int)level);
        float p[3] = {(((float)x + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f, (((float)y + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f,
                      (((float)z + 0.5f) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f};
        float voxel_radius = 0.5f * SQRT3_ * sc / NERF_GRIDSIZE;
        int count = 0;
        for (uint32_t j = 0; j < n_images; ++j) {
            const float* m = xforms + 12 * j; /* column-major 3x4: col c = m[3c..3c+2] */
            float pl[3] = {p[0] - m[9], p[1] - m[10], p[2] - m[11]};
            float cx = pl[0] * m[0] + (pl[1] * m[1] + pl[2] * m[2]); /* Eigen redux association */
            float cy = pl[0] * m[3] + (pl[1] * m[4] + pl[2] * m[5]);
            float cz = pl[0] * m[6] + (pl[1] * m[7] + pl[2] * m[8]);
            if (cz > 0.f) {
                if (fabsf(cx) - voxel_radius < cz / focal[2 * j] * half_resx && fabsf(cy) - voxel_radius < cz / focal[2 * j + 1] * half_resy) {
                    count++; break;
                }
            }
        }
        if ((grid[i] < 0) != (count <= 0)) grid[i] = (count > 0) ? 0.f : -1.f;
    }
}
/* generate_grid_samples_nerf_nonuniform.h:3-36 */
void orc_generate_grid_samples(uint32_t n_elements, uint64_t rng_state, uint64_t rng_inc, uint32_t step, float aabb_lo,
                               float aabb_hi, const float* grid_in, float* positions, uint32_t* indices,
                               uint32_t n_cascades, float thresh) {
    const uint32_t G3 = NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE;
    float diag = aabb_hi - aabb_lo;
#pragma omp parallel for schedule(static)
    for (int64_t ii = 0; ii < (int64_t)n_elements; ++ii) {
        uint32_t i = (uint32_t)ii;
        orc_pcg32 rng = {rng_state, rng_inc};
        pcg_advance(&rng, (int64_t)(uint32_t)(i * 4u));
        uint32_t level = (uint32_t)(pcg_next_float(&rng) * n_cascades) % n_cascades;
        uint32_t idx = 0;
        for (uint32_t j = 0; j < 10; ++j) {
            idx = ((i + step * n_elements) * 56924617u + j * 19349663u + 96925573u) % G3;
            idx += level * G3;
            if (grid_in[idx] > thresh) break;
        }
        uint32_t pos_idx = idx % G3;
        uint32_t x = morton3D_invert(pos_idx >> 0), y = morton3D_invert(pos_idx >> 1), z = morton3D_invert(pos_idx >> 2);
        float r0 = pcg_next_float(&rng), r1 = pcg_next_float(&rng), r2 = pcg_next_float(&rng);
        float sc = scalbnf(1.0f, (int)level);
        float p[3] = {(((float)x + r0) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f, (((float)y + r1) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f,
                      (((float)z + r2) / NERF_GRIDSIZE - 0.5f) * sc + 0.5f};
        positions[3 * (size_t)i] = (p[0] - aabb_lo) / diag;
        positions[3 * (size_t)i + 1] = (p[1] - aabb_lo) / diag;
        positions[3 * (size_t)i + 2] = (p[2] - aabb_lo) / diag;
        indices[i] = idx;
    }
}
/* splat_grid_samples_nerf_max_nearest_neighbor.h:4-23 ; mlp_out stride 1 (density_grid_sampler.py:53) */
void orc_splat(uint32_t n, const uint32_t* indices, const void* mlp_out, int is_half, float* grid_tmp) {
    for (uint32_t i = 0; i < n; ++i) {
        float v = is_half ? h2f(((const half_t*)mlp_out)[i]) : ((const float*)mlp_out)[i];
        float thick = expf(v) * (SQRT3_ / NERF_STEPS);
        uint32_t u; memcpy(&u, &thick, 4);
        uint32_t* cell = (uint32_t*)&grid_tmp[indices[i]];
        if (u > *cell) *cell = u;
    }
}
/* ema_grid_samples_nerf.h:3-26 */
void orc_ema(uint32_t n, float decay, float* grid, const float* grid_tmp) {
    for (uint32_t i = 0; i < n; ++i) {
        float prev = grid[i];
        grid[i] = (prev < 0.f) ? prev : fmaxf(prev * decay, grid_tmp[i]);
    }
}
/* update_bitfield.py:13-37: mean over cascade 0 of max(v,0)/n, then grid_to_bitfield + 4 max-pools */
float orc_grid_mean(const float* grid) {
    const uint32_t G3 = NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE;
    double s = 0;
    for (uint32_t i = 0; i < G3; ++i) s += (double)(fmaxf(grid[i], 0.f) / G3);
    return (float)s;
}
void orc_update_bitfield(const float* grid, float mean, uint32_t cascades, uint8_t* bitfield) {
    const uint32_t G3 = NERF_GRIDSIZE * NERF_GRIDSIZE * NERF_GRIDSIZE;
    float thresh = 0.01f < mean ? 0.01f : mean;
    for (uint32_t i = 0; i < G3 / 8 * cascades; ++i) {
        uint8_t bits = 0;
        for (int j = 0; j < 8; ++j) bits |= grid[(size_t)i * 8 + j] > thresh ? (uint8_t)(1 << j) : 0;
        bitfield[i] = bits;
    }
    for (uint32_t level = 1; level < cascades; ++level) {
        const uint8_t* prev = bitfield + (size_t)G3 * (level - 1) / 8;
        uint8_t* next = bitfield + (size_t)G3 * level / 8;
        for (uint32_t i = 0; i < G3 / 64; ++i) {
            uint8_t bits = 0;
            for (int j = 0; j < 8; ++j) bits |= prev[(size_t)i * 8 + j] > 0 ? (uint8_t)(1 << j) : 0;
            uint32_t x = morton3D_invert(i >> 0) + NERF_GRIDSIZE / 8, y = morton3D_invert(i >> 1) + NERF_GRIDSIZE / 8,
                     z = morton3D_invert(i >> 2) + NERF_GRIDSIZE / 8;
            next[morton3D(x, y, z)] |= bits;
        }
    }
}

/* ------------------------------------------------------------------------------------------------
 * N1: Adam + EMA (PARITY UNPINNED -- Jittor is not in the reference tree).  Restated from
 *     optims/adam.py:8-16 (jt.nn.Adam: step_size = lr*sqrt(1-b2^n)/(1-b1^n); p -= m*step_size/(sqrt(v)+eps)),
 *     optims/expdecay.py:20-25, optims/ema.py:26-37 (EMA overwrites the live parameters).
 *     State fp32 (deliberate, documented deviation for fp16 params); param stored fp16 or fp32.
 * ---------------------------------------------------------------------------------------------- */
void orc_adam_ema(uint64_t n, void* param, int is_half, const float* grad, float* m, float* v, float* master,
                  float lr, float b1, float b2, float eps, uint32_t step /*1-based*/, float ema_decay) {
    /* `master` is the EMA optimizer's `values` buffer (ema.py:16-19, a copy of the params), kept in fp32: after
     * every ema_step the live parameter equals it (ema.py:33-36), so it doubles as the fp32 master weight. */
    double n1 = 1.0 - pow((double)b1, (double)step), n2 = 1.0 - pow((double)b2, (double)step);
    float step_size = (float)(lr * sqrt(n2) / n1);
    float debias_old = (float)(1.0 - pow((double)ema_decay, (double)step - 1.0));
    float debias_new = (float)(1.0 / (1.0 - pow((double)ema_decay, (double)step)));
    for (uint64_t i = 0; i < n; ++i) {
        float p = master[i];
        float g = grad[i];
        m[i] = b1 * m[i] + (1 - b1) * g;
        v[i] = b2 * v[i] + (1 - b2) * g * g;
        p = p - m[i] * step_size / (sqrtf(v[i]) + eps);
        float pe = ((1 - ema_decay) * p + ema_decay * master[i] * debias_old) * debias_new;
        master[i] = pe;
        if (is_half) ((half_t*)param)[i] = f2h(pe); else ((float*)param)[i] = pe;
    }
}

/* ------------------------------------------------------------------------------------------------
 * N2: ray generation (dataset/dataset.py:172-188).  xforms column-major 3x4.  float tolerance only.
 * ---------------------------------------------------------------------------------------------- */
void orc_raygen(uint32_t n, const uint32_t* pix_index /* global pixel ids */, uint32_t W, uint32_t H, const float* xforms,
                const float* focal /* (n_img,2) */, const float* principal /* (n_img,2) */, uint32_t* img_id, float* rays_o,
                float* rays_d) {
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t id = pix_index[i] / (H * W), off = pix_index[i] % (H * W);
        const float* m = xforms + 12 * id;
        float x = ((off % W) + 0.5f) / W, y = ((off / W) + 0.5f) / H;
        float dx = (x - principal[2 * id]) * W / focal[2 * id], dy = (y - principal[2 * id + 1]) * H / focal[2 * id + 1], dz = 1.0f;
        float d[3] = {m[0] * dx + m[3] * dy + m[6] * dz, m[1] * dx + m[4] * dy + m[7] * dz, m[2] * dx + m[5] * dy + m[8] * dz};
        float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        nrm = nrm > 1e-12f ? nrm : 1e-12f;
        img_id[i] = id;
        rays_o[3 * i] = m[9]; rays_o[3 * i + 1] = m[10]; rays_o[3 * i + 2] = m[11];
        rays_d[3 * i] = d[0] / nrm; rays_d[3 * i + 1] = d[1] / nrm; rays_d[3 * i + 2] = d[2] / nrm;
    }
}
