// Lattice smoothing before marching cubes: the reference's --mcube_smooth (tools/extract_mesh.py:27-31,74-78), which calls PyMCubes'
// smooth(sigma) and marches the result at 0.  The contract is restated in DESIGN.md section 7; two methods:
//  - constrained (Lempitsky 2010): the signed distance D of the inside set from an exact Euclidean distance transform, then, on the
//    band |D| < 4, a Jacobi solve in fp64 that lowers the sum of squared second differences while keeping every voxel on its side;
//  - gaussian: a separable sigma-3 Gaussian of f - 0.5 in fp64 (scipy's gaussian_filter with mode 'reflect').
// Every result is bit-reproducible: the EDT is integer, every sum runs in a fixed order, and the band kernels run on a fixed grid
// (independent of the device's SM count), so the energies that decide when the solve stops are the same on every run.
#include <cmath>

#include "ngp_common.cuh"
#include "mesh_scan.cuh"

namespace {

constexpr uint32_t LINE_THREADS = 128;                  // one CTA per lattice line (n <= 1024 values in shared memory)
constexpr uint32_t BAND_THREADS = 256, BAND_GRID = 1024;  // fixed grid of the band loops: the energy partials do not depend on the device
constexpr int32_t EDT_INF = 0x7fffffff;                 // squared distance of a voxel with no feature voxel in reach (yet)
constexpr double BAND_RADIUS = 4.0;
constexpr uint32_t CHECK_EVERY = 10;                    // energy test every 10 iterations
constexpr double REL_TOL = 1e-6;
constexpr uint32_t AUTO_MAX_N = 512;                    // method 0: constrained up to 512^3, gaussian above
constexpr int GAUSS_R = 12;                             // sigma 3, truncate 4: int(4 * 3 + 0.5) taps on each side

struct SmoothState {
    uint32_t n_vars, iters, stop, pad;
    double e_prev;                                      // energy at the previous check (E(x0) before the first)
};

// lattice line L along `axis`: first point and stride (row (i*n + j)*n + k)
__device__ __forceinline__ void line_of(uint32_t n, uint32_t axis, uint32_t L, uint32_t& base, uint32_t& stride) {
    if (axis == 2) { base = L * n; stride = 1; }                              // L = i*n + j
    else if (axis == 1) { base = (L / n) * n * n + L % n; stride = n; }       // L = i*n + k
    else { base = L; stride = n * n; }                                        // L = j*n + k
}

// ---- exact Euclidean distance transform (Felzenszwalb-Huttenlocher, separable on int32 squared distances) ---------------------------
// g0: 0 on outside voxels (the distance of an inside voxel to the outside), g1: 0 on inside voxels; INF elsewhere.
__global__ void edt_init_kernel(uint32_t n3, const float* __restrict__ f, int32_t* __restrict__ g0, int32_t* __restrict__ g1) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n3) return;
    const bool in = f[p] > 0.f;
    g0[p] = in ? EDT_INF : 0;
    g1[p] = in ? 0 : EDT_INF;
}

// One line of both transforms (blockIdx.y picks g0 / g1) in place: g[p] <- min_q g[q] + (p - q)^2.  Thread 0 builds the lower envelope of
// the parabolas (boundaries z kept as exact fractions zn / zd, zd > 0); every thread then finds its parabola by bisection.
__global__ void __launch_bounds__(LINE_THREADS) edt_line_kernel(uint32_t n, uint32_t axis, int32_t* __restrict__ g0, int32_t* __restrict__ g1) {
    extern __shared__ int32_t sm_edt[];
    int32_t *g = sm_edt, *v = sm_edt + n, *zn = sm_edt + 2 * n, *zd = sm_edt + 3 * n;
    __shared__ int32_t n_env;
    int32_t* buf = blockIdx.y ? g1 : g0;
    uint32_t base, stride;
    line_of(n, axis, blockIdx.x, base, stride);
    for (uint32_t p = threadIdx.x; p < n; p += LINE_THREADS) g[p] = buf[base + p * stride];
    __syncthreads();
    if (threadIdx.x == 0) {
        int32_t k = -1;
        for (int32_t q = 0; q < (int32_t)n; ++q) {
            if (g[q] == EDT_INF) continue;
            const int32_t hq = g[q] + q * q;
            int32_t num = 0, den = 1;
            while (k >= 0) {
                const int32_t r = v[k];
                num = hq - (g[r] + r * r);                                    // parabolas r and q meet at num / den
                den = 2 * (q - r);
                if (k == 0 || (int64_t)num * zd[k] > (int64_t)zn[k] * den) break;   // right of where r's segment starts: r stays
                --k;
            }
            ++k;
            v[k] = q; zn[k] = num; zd[k] = den;                               // (z[0] is -inf and never read)
        }
        n_env = k + 1;
    }
    __syncthreads();
    const int32_t K = n_env;
    for (uint32_t p = threadIdx.x; p < n; p += LINE_THREADS) {
        int32_t out = EDT_INF;
        if (K > 0) {
            int32_t lo = 0, hi = K - 1;                                       // the last segment starting at or left of p
            while (lo < hi) {
                const int32_t mid = (lo + hi + 1) >> 1;
                if ((int64_t)zn[mid] <= (int64_t)p * zd[mid]) lo = mid; else hi = mid - 1;
            }
            const int32_t r = v[lo], d = (int32_t)p - r;
            out = g[r] + d * d;
        }
        buf[base + p * stride] = out;
    }
}

// signed squared distance s (+ inside, - outside) -> D = +-(sqrt(|s|) - 0.5); +-1 when the other class is empty
__device__ __forceinline__ double sdist(int32_t s) {
    const int32_t k = s < 0 ? -s : s;
    const double d = k == EDT_INF ? 1.0 : sqrt((double)k) - 0.5;
    return s < 0 ? -d : d;
}
__device__ __forceinline__ bool in_band(int32_t s) {
    const int32_t k = s < 0 ? -s : s;
    return k != EDT_INF && sqrt((double)k) - 0.5 < BAND_RADIUS;
}

// combines the two transforms into s (in place of g0), writes D to field_out and the band flags (in place of g1)
__global__ void smooth_mark_kernel(uint32_t n3, const float* __restrict__ f, int32_t* g0_s, int32_t* g1_mark, float* __restrict__ field_out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n3) return;
    const int32_t s = f[p] > 0.f ? g0_s[p] : -g1_mark[p];
    g0_s[p] = s;
    g1_mark[p] = in_band(s);
    field_out[p] = (float)sdist(s);
}

// per band variable c = idx[p]: x0 = D, its one finite bound (sign bit set = an upper bound), and the six neighbours (-1: outside the
// lattice or the band) in the order -i, +i, -j, +j, -k, +k
__global__ void smooth_band_kernel(uint32_t n, const int32_t* __restrict__ s, const uint32_t* __restrict__ idx, int32_t* __restrict__ nb,
                                   double* __restrict__ x, double* __restrict__ bnd) {
    const uint32_t n3 = n * n * n, p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n3 || !in_band(s[p])) return;
    const uint32_t c = idx[p], co[3] = {p / (n * n), (p / n) % n, p % n}, st[3] = {n * n, n, 1u};
#pragma unroll
    for (uint32_t a = 0; a < 3; ++a) {
        nb[6 * (size_t)c + 2 * a] = co[a] > 0 && in_band(s[p - st[a]]) ? (int32_t)idx[p - st[a]] : -1;
        nb[6 * (size_t)c + 2 * a + 1] = co[a] + 1 < n && in_band(s[p + st[a]]) ? (int32_t)idx[p + st[a]] : -1;
    }
    const double d = sdist(s[p]);
    x[c] = d;
    bnd[c] = fabs(d) < 1.0 ? (d > 0 ? 0.0 : -0.0) : d;                       // a finite bound below 1 in size becomes 0
}

__global__ void smooth_state_kernel(SmoothState* st, uint32_t max_iters) {
    st->iters = max_iters;
    st->stop = 0;
    st->e_prev = 0.0;
}

// sum over the block in a fixed order (blockDim.x = 32 * w, w <= 32); the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double sh[32];
#pragma unroll
    for (uint32_t o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (uint32_t w = 0; w < (blockDim.x >> 5); ++w) t += sh[w];
    return t;
}

// q = Qx: q_a(c) = (m_a(c) - 2) x_c + the counted neighbours along a; with `energy`, part[block] = sum of q^2 over the block's variables
__global__ void __launch_bounds__(BAND_THREADS) smooth_q_kernel(const SmoothState* __restrict__ st, const int32_t* __restrict__ nb,
                                                                const double* __restrict__ x, double* __restrict__ q, double* __restrict__ part,
                                                                int energy) {
    if (st->stop) return;
    const uint32_t M = st->n_vars;
    double e = 0.0;
    for (uint32_t c = blockIdx.x * BAND_THREADS + threadIdx.x; c < M; c += BAND_GRID * BAND_THREADS) {
        const double xc = x[c];
#pragma unroll
        for (uint32_t a = 0; a < 3; ++a) {
            const int32_t lo = nb[6 * (size_t)c + 2 * a], hi = nb[6 * (size_t)c + 2 * a + 1];
            double qa = (double)((int32_t)(lo < 0) + (int32_t)(hi < 0) - 2) * xc;
            if (lo >= 0) qa += x[lo];
            if (hi >= 0) qa += x[hi];
            q[3 * (size_t)c + a] = qa;
            e += qa * qa;
        }
    }
    if (energy) {
        const double t = block_sum(e);
        if (threadIdx.x == 0) part[blockIdx.x] = t;
    }
}

// E = sum(part) / 2 of x_t in a fixed order; t = 0 records E(x0), every later check stops the loop (at t) on a relative decrease below
// stop_ratio.  A 0/0 ratio is NaN and does not stop it.
__global__ void __launch_bounds__(BAND_GRID) smooth_check_kernel(SmoothState* st, const double* __restrict__ part, uint32_t t, double stop_ratio) {
    const bool stopped = st->stop != 0;
    const double E = 0.5 * block_sum(part[threadIdx.x]);
    if (threadIdx.x != 0 || stopped) return;
    if (t == 0) {
        st->e_prev = E;
    } else if ((st->e_prev - E) / st->e_prev < stop_ratio) {
        st->stop = 1;
        st->iters = t;
    } else {
        st->e_prev = E;
    }
}

// x <- clamp(x/2 + xhat/2), xhat = -(Ax - diag(A) x) / diag(A), Ax = Q^T q gathered from the neighbours' q; a variable with no counted
// neighbour (diagonal 0) keeps x0
__global__ void __launch_bounds__(BAND_THREADS) smooth_update_kernel(const SmoothState* __restrict__ st, const int32_t* __restrict__ nb,
                                                                     const double* __restrict__ q, const double* __restrict__ bnd, double* __restrict__ x) {
    if (st->stop) return;
    const uint32_t M = st->n_vars;
    for (uint32_t c = blockIdx.x * BAND_THREADS + threadIdx.x; c < M; c += BAND_GRID * BAND_THREADS) {
        double ax = 0.0;
        int32_t d = 0;
#pragma unroll
        for (uint32_t a = 0; a < 3; ++a) {
            const int32_t lo = nb[6 * (size_t)c + 2 * a], hi = nb[6 * (size_t)c + 2 * a + 1];
            const int32_t m = (int32_t)(lo < 0) + (int32_t)(hi < 0);
            ax += (double)(m - 2) * q[3 * (size_t)c + a];
            if (lo >= 0) ax += q[3 * (size_t)lo + a];
            if (hi >= 0) ax += q[3 * (size_t)hi + a];
            d += (m - 2) * (m - 2) + 2 - m;
        }
        if (d == 0) continue;
        const double xc = x[c], dd = (double)d;
        const double xh = -(ax - dd * xc) / dd;
        const double xn = 0.5 * xh + 0.5 * xc, b = bnd[c];
        x[c] = signbit(b) ? fmin(xn, b) : fmax(xn, b);
    }
}

__global__ void smooth_scatter_kernel(uint32_t n3, const int32_t* __restrict__ s, const uint32_t* __restrict__ idx, const double* __restrict__ x,
                                      float* __restrict__ field_out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n3 && in_band(s[p])) field_out[p] = (float)x[idx[p]];
}

// ---- Gaussian --------------------------------------------------------------------------------------------------------------------
struct GaussWeights { double w[GAUSS_R + 1]; };      // w[j] = w[-j]

// mode 'reflect' (d c b a | a b c d | d c b a): period 2n
__device__ __forceinline__ int32_t reflect(int32_t i, int32_t n) {
    i %= 2 * n;
    if (i < 0) i += 2 * n;
    return i < n ? i : 2 * n - 1 - i;
}

// one line along `axis`, in place in buf; the first pass reads f - 0.5, the last writes fp32.  The sum runs as scipy's symmetric
// correlate1d does: centre first, then the pairs from the outermost in.
template <bool FIRST, bool LAST>
__global__ void __launch_bounds__(LINE_THREADS) gauss_line_kernel(uint32_t n, uint32_t axis, const float* __restrict__ f, double* buf,
                                                                  float* __restrict__ out, GaussWeights w) {
    extern __shared__ double sm_line[];
    uint32_t base, stride;
    line_of(n, axis, blockIdx.x, base, stride);
    for (uint32_t p = threadIdx.x; p < n; p += LINE_THREADS) sm_line[p] = FIRST ? (double)f[base + p * stride] - 0.5 : buf[base + p * stride];
    __syncthreads();
    for (uint32_t p = threadIdx.x; p < n; p += LINE_THREADS) {
        double acc = sm_line[p] * w.w[0];
#pragma unroll
        for (int32_t j = GAUSS_R; j > 0; --j)
            acc += (sm_line[reflect((int32_t)p - j, (int32_t)n)] + sm_line[reflect((int32_t)p + j, (int32_t)n)]) * w.w[j];
        if (LAST) out[base + p * stride] = (float)acc;
        else buf[base + p * stride] = acc;
    }
}

// scipy's _gaussian_kernel1d(3, 0, 12): exp(-0.5 / 9 * j^2) over the sum, which numpy forms pairwise (eight running sums, then the rest)
GaussWeights gauss_weights() {
    double phi[2 * GAUSS_R + 1];
    for (int j = -GAUSS_R; j <= GAUSS_R; ++j) phi[j + GAUSS_R] = std::exp(-0.5 / 9.0 * (double)(j * j));
    double r[8];
    for (int i = 0; i < 8; ++i) r[i] = phi[i];
    int i = 8;
    for (; i < 2 * GAUSS_R + 1 - (2 * GAUSS_R + 1) % 8; i += 8)
        for (int k = 0; k < 8; ++k) r[k] += phi[i + k];
    double sum = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < 2 * GAUSS_R + 1; ++i) sum += phi[i];
    GaussWeights w;
    for (int j = 0; j <= GAUSS_R; ++j) w.w[j] = phi[GAUSS_R + j] / sum;
    return w;
}

// ---- workspace ----------------------------------------------------------------------------------------------------------------------
inline uint64_t al(uint64_t b) { return (b + 255) & ~uint64_t(255); }
inline uint32_t blocks(uint64_t n, uint32_t per) { return (uint32_t)((n + per - 1) / per); }
inline uint32_t pick_method(uint32_t n, uint32_t method) { return method ? method : (n <= AUTO_MAX_N ? 1u : 2u); }

struct SmoothWs {
    int32_t *s, *nb; uint32_t *idx, *bsum; SmoothState* st; double *part, *x, *q, *bnd, *g;
    // constrained: s, idx (4 n^3 each), bsum, state, partials, then per possible variable (n^3 at most) nb (24), x (8), q (24), bnd (8);
    // gaussian: one fp64 lattice (8 n^3)
    static uint64_t layout(uint32_t n, uint32_t method, uint8_t* w, SmoothWs* o) {
        const uint64_t n3 = (uint64_t)n * n * n;
        uint64_t at = 0;
        auto take = [&](uint64_t bytes) { uint8_t* p = w ? w + at : nullptr; at += al(bytes); return p; };
        SmoothWs r{};
        if (method == 1) {
            r.s = (int32_t*)take(4 * n3); r.idx = (uint32_t*)take(4 * n3); r.bsum = (uint32_t*)take(4 * (uint64_t)blocks(n3, ngp_mesh::SCAN_BLOCK));
            r.st = (SmoothState*)take(sizeof(SmoothState)); r.part = (double*)take(8 * BAND_GRID);
            r.nb = (int32_t*)take(24 * n3); r.x = (double*)take(8 * n3); r.q = (double*)take(24 * n3); r.bnd = (double*)take(8 * n3);
        } else {
            r.g = (double*)take(8 * n3);
        }
        if (o) *o = r;
        return at;
    }
};

int check_smooth_args(const char* fn, uint32_t n, uint32_t method) {
    NGP_REQUIRE(n >= 2 && n <= 1024, std::string(fn) + ": resolution n must be in [2, 1024], got " + std::to_string(n));
    NGP_REQUIRE(method <= 2, std::string(fn) + ": method must be 0 (auto), 1 (constrained) or 2 (gaussian), got " + std::to_string(method));
    return 0;
}

int smooth_constrained(cudaStream_t s, uint32_t n, const float* field, uint32_t max_iters, const SmoothWs& w, float* field_out, uint32_t* info) {
    const uint32_t n3 = n * n * n, nb3 = blocks(n3, 256);
    const size_t edt_smem = 4 * sizeof(int32_t) * n;
    edt_init_kernel<<<nb3, 256, 0, s>>>(n3, field, w.s, (int32_t*)w.idx);
    NGP_LAUNCH_CHECK();
    for (uint32_t axis = 3; axis-- > 0;) {                                   // along k, then j, then i
        edt_line_kernel<<<dim3(n * n, 2), LINE_THREADS, edt_smem, s>>>(n, axis, w.s, (int32_t*)w.idx);
        NGP_LAUNCH_CHECK();
    }
    smooth_mark_kernel<<<nb3, 256, 0, s>>>(n3, field, w.s, (int32_t*)w.idx, field_out);
    NGP_LAUNCH_CHECK();
    smooth_state_kernel<<<1, 1, 0, s>>>(w.st, max_iters);
    NGP_LAUNCH_CHECK();
    if (int rc = ngp_mesh::scan_u32(s, w.idx, n3, w.bsum, &w.st->n_vars)) return rc;
    smooth_band_kernel<<<nb3, 256, 0, s>>>(n, w.s, w.idx, w.nb, w.x, w.bnd);
    NGP_LAUNCH_CHECK();
    const double stop_ratio = 1.0 - std::pow(1.0 - REL_TOL, (double)CHECK_EVERY);
    for (uint32_t t = 1; t <= max_iters; ++t) {                              // no host sync: a stop flag on the device ends the work
        const bool check = (t - 1) % CHECK_EVERY == 0;
        smooth_q_kernel<<<BAND_GRID, BAND_THREADS, 0, s>>>(w.st, w.nb, w.x, w.q, w.part, check);
        NGP_LAUNCH_CHECK();
        if (check) {
            smooth_check_kernel<<<1, BAND_GRID, 0, s>>>(w.st, w.part, t - 1, stop_ratio);
            NGP_LAUNCH_CHECK();
        }
        smooth_update_kernel<<<BAND_GRID, BAND_THREADS, 0, s>>>(w.st, w.nb, w.q, w.bnd, w.x);
        NGP_LAUNCH_CHECK();
    }
    smooth_scatter_kernel<<<nb3, 256, 0, s>>>(n3, w.s, w.idx, w.x, field_out);
    NGP_LAUNCH_CHECK();
    SmoothState st;
    NGP_CHECK_CUDA(cudaMemcpyAsync(&st, w.st, sizeof(st), cudaMemcpyDeviceToHost, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    info[1] = st.iters;
    info[2] = st.n_vars;
    return 0;
}

int smooth_gaussian(cudaStream_t s, uint32_t n, const float* field, const SmoothWs& w, float* field_out) {
    const GaussWeights gw = gauss_weights();
    const size_t smem = sizeof(double) * n;
    gauss_line_kernel<true, false><<<n * n, LINE_THREADS, smem, s>>>(n, 0, field, w.g, nullptr, gw);
    NGP_LAUNCH_CHECK();
    gauss_line_kernel<false, false><<<n * n, LINE_THREADS, smem, s>>>(n, 1, nullptr, w.g, nullptr, gw);
    NGP_LAUNCH_CHECK();
    gauss_line_kernel<false, true><<<n * n, LINE_THREADS, smem, s>>>(n, 2, nullptr, w.g, field_out, gw);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" {

int ngp_mesh_smooth_workspace_bytes(uint32_t n, uint32_t method, uint64_t* bytes_out) {
    if (int rc = check_smooth_args("ngp_mesh_smooth_workspace_bytes", n, method)) return rc;
    NGP_REQUIRE(bytes_out, "ngp_mesh_smooth_workspace_bytes: bytes_out is required");
    *bytes_out = SmoothWs::layout(n, pick_method(n, method), nullptr, nullptr);
    return 0;
}

int ngp_mesh_smooth(void* stream, uint32_t n, const float* field, uint32_t method, uint32_t max_iters, void* workspace, uint64_t workspace_bytes,
                    float* field_out, uint32_t* info_host) {
    if (int rc = check_smooth_args("ngp_mesh_smooth", n, method)) return rc;
    NGP_REQUIRE(field && workspace && field_out && info_host, "ngp_mesh_smooth: field, workspace, field_out and info_host are required");
    NGP_REQUIRE(field_out != field, "ngp_mesh_smooth: field_out must be a separate buffer from field");
    const uint32_t m = pick_method(n, method);
    SmoothWs w;
    const uint64_t need = SmoothWs::layout(n, m, (uint8_t*)workspace, &w);
    NGP_REQUIRE(workspace_bytes >= need, "ngp_mesh_smooth: the workspace has " + std::to_string(workspace_bytes) + " bytes, method " +
                std::to_string(m) + " at n = " + std::to_string(n) + " needs " + std::to_string(need));
    cudaStream_t s = (cudaStream_t)stream;
    info_host[0] = m;
    info_host[1] = info_host[2] = 0;
    return m == 1 ? smooth_constrained(s, n, field, max_iters, w, field_out, info_host) : smooth_gaussian(s, n, field, w, field_out);
}

}  // extern "C"
