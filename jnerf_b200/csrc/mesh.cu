// Mesh extraction (tools/extract_mesh.py:42-106 of the reference): marching cubes on the density lattice, the largest
// edge-connected component and area-weighted vertex normals, all on the device.  The reference runs PyMCubes and Open3D on the host.
//
// Every result is independent of the launch configuration and of scheduling: vertices are numbered in lattice-edge order, triangles
// in cell order, component labels are the smallest triangle of their cluster, and every floating-point sum runs in a fixed order.
// Built with -fmad=false (like sampler.cu): the interpolation and the cross products match the oracle bit for bit.
#include "ngp_common.cuh"
#include "mc_table.cuh"
#include "mesh_scan.cuh"

using ngp_mesh::scan_u32;

namespace {

constexpr uint32_t MC_THREADS = 256, MC_PPT = 8, MC_BLOCK = MC_THREADS * MC_PPT;   // lattice points per block (8 consecutive per thread)
constexpr uint32_t SC_THREADS = 256, SC_PPT = 8, SC_BLOCK = SC_THREADS * SC_PPT;   // elements per block of the u32 scans
static_assert(SC_BLOCK == ngp_mesh::SCAN_BLOCK, "mesh_scan.cuh states the scan's block size");
constexpr uint32_t TOP_THREADS = 1024;                                              // the single-CTA scan over block sums
constexpr uint32_t LOCAL_BITS = 13;   // per point: vertex offset inside its block (< 3 * MC_BLOCK = 6144) | crossing mask << 13

__device__ const int8_t g_mc_tri[256][3 * NGP_MC_MAX_TRIS] = NGP_MC_TRI_TABLE;
__device__ const uint8_t g_mc_ntri[256] = NGP_MC_TRI_COUNT;

// exclusive scan over the block (blockDim.x a multiple of 32, at most 1024); sh: 32 elements; total = the block's sum
template <class T>
__device__ __forceinline__ T block_excl_scan(T v, T* sh, T& total) {
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T x = v;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[w] = x;
    __syncthreads();
    if (w == 0) {
        T s = lane < nw ? sh[lane] : T(0);
#pragma unroll
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < nw) sh[lane] = s;
    }
    __syncthreads();
    const T r = (w ? sh[w - 1] : T(0)) + x - v;
    total = sh[nw - 1];
    __syncthreads();
    return r;
}

// exclusive scan of cnt[0..nb) into base (in place allowed), one CTA; the sum goes to *total
template <class T>
__device__ void top_scan(const uint32_t* cnt, T* base, uint32_t nb, T* total) {
    __shared__ T sh[32];
    const uint32_t chunk = (nb + TOP_THREADS - 1) / TOP_THREADS, lo = min(threadIdx.x * chunk, nb), hi = min(lo + chunk, nb);
    T s = 0;
    for (uint32_t i = lo; i < hi; ++i) s += cnt[i];
    T tot;
    T run = block_excl_scan<T>(s, sh, tot);
    for (uint32_t i = lo; i < hi; ++i) {
        const T c = cnt[i];
        base[i] = run;
        run += c;
    }
    if (threadIdx.x == 0) *total = tot;
}

// ---- marching cubes ------------------------------------------------------------------------------------
__device__ __forceinline__ bool inside(float v, float iso) { return v > iso; }

// crossing edges (bit axis) of lattice point p = (i, j, k)
__device__ __forceinline__ uint32_t edge_mask(const float* __restrict__ f, uint32_t n, float iso, uint32_t p, uint32_t i, uint32_t j, uint32_t k) {
    const bool a = inside(f[p], iso);
    uint32_t m = 0;
    if (i + 1 < n && a != inside(f[p + n * n], iso)) m |= 1u;
    if (j + 1 < n && a != inside(f[p + n], iso)) m |= 2u;
    if (k + 1 < n && a != inside(f[p + 1], iso)) m |= 4u;
    return m;
}
// case of the cell whose lowest corner is p, or 0 when p is on the upper boundary (no cell)
__device__ __forceinline__ uint32_t cell_case(const float* __restrict__ f, uint32_t n, float iso, uint32_t p, uint32_t i, uint32_t j, uint32_t k) {
    if (i + 1 >= n || j + 1 >= n || k + 1 >= n) return 0;
    uint32_t cs = 0;
#pragma unroll
    for (uint32_t c = 0; c < 8; ++c) cs |= (uint32_t)inside(f[p + (c & 1) * n * n + ((c >> 1) & 1) * n + ((c >> 2) & 1)], iso) << c;
    return cs;
}

// Per block of MC_BLOCK points: the crossing mask and block-local vertex offset of every point, and the block's vertex and triangle
// counts.
__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(uint32_t n, const float* __restrict__ f, float iso, uint16_t* __restrict__ local,
                                                              uint32_t* __restrict__ bcnt_v, uint32_t* __restrict__ bcnt_t) {
    __shared__ uint32_t sh[32];
    const uint32_t n3 = n * n * n, p0 = blockIdx.x * MC_BLOCK + threadIdx.x * MC_PPT;
    uint32_t masks = 0, nv = 0, nt = 0;
#pragma unroll
    for (uint32_t q = 0; q < MC_PPT; ++q) {
        const uint32_t p = p0 + q;
        if (p >= n3) break;
        const uint32_t k = p % n, j = (p / n) % n, i = p / (n * n);
        const uint32_t m = edge_mask(f, n, iso, p, i, j, k);
        masks |= m << (3 * q);
        nv += __popc(m);
        nt += g_mc_ntri[cell_case(f, n, iso, p, i, j, k)];
    }
    uint32_t tot_v, tot_t;
    uint32_t off = block_excl_scan<uint32_t>(nv, sh, tot_v);
    block_excl_scan<uint32_t>(nt, sh, tot_t);
#pragma unroll
    for (uint32_t q = 0; q < MC_PPT; ++q) {
        const uint32_t p = p0 + q;
        if (p >= n3) break;
        const uint32_t m = (masks >> (3 * q)) & 7u;
        local[p] = (uint16_t)(off | (m << LOCAL_BITS));
        off += __popc(m);
    }
    if (threadIdx.x == 0) { bcnt_v[blockIdx.x] = tot_v; bcnt_t[blockIdx.x] = tot_t; }
}

__global__ void __launch_bounds__(TOP_THREADS) mc_scan_kernel(const uint32_t* __restrict__ bcnt_v, const uint32_t* __restrict__ bcnt_t,
                                                              uint64_t* __restrict__ base_v, uint64_t* __restrict__ base_t, uint32_t nb,
                                                              uint64_t* __restrict__ totals) {
    top_scan<uint64_t>(bcnt_v, base_v, nb, totals);
    __syncthreads();
    top_scan<uint64_t>(bcnt_t, base_t, nb, totals + 1);
}

// vertex index of lattice edge (point pp, axis a), which crosses
__device__ __forceinline__ uint32_t edge_vertex(const uint16_t* __restrict__ local, const uint64_t* __restrict__ base_v, uint32_t pp, uint32_t a) {
    const uint32_t L = local[pp];
    return (uint32_t)base_v[pp / MC_BLOCK] + (L & ((1u << LOCAL_BITS) - 1u)) + __popc((L >> LOCAL_BITS) & ((1u << a) - 1u));
}

// Vertices (PLY frame: lattice position / N, first two columns swapped) and triangles of every block, at the scanned offsets.
__global__ void __launch_bounds__(MC_THREADS) mc_emit_kernel(uint32_t n, const float* __restrict__ f, float iso, const uint16_t* __restrict__ local,
                                                             const uint64_t* __restrict__ base_v, const uint64_t* __restrict__ base_t,
                                                             float* __restrict__ verts, int32_t* __restrict__ tris) {
    __shared__ int8_t s_tri[256][3 * NGP_MC_MAX_TRIS];
    __shared__ uint32_t sh[32];
    for (uint32_t i = threadIdx.x; i < 256 * 3 * NGP_MC_MAX_TRIS; i += MC_THREADS) (&s_tri[0][0])[i] = (&g_mc_tri[0][0])[i];
    const uint32_t n3 = n * n * n, p0 = blockIdx.x * MC_BLOCK + threadIdx.x * MC_PPT;
    const float fn = (float)n;
    uint8_t cases[MC_PPT];
    uint32_t nt = 0;
#pragma unroll
    for (uint32_t q = 0; q < MC_PPT; ++q) {
        const uint32_t p = p0 + q;
        cases[q] = 0;
        if (p >= n3) continue;
        const uint32_t k = p % n, j = (p / n) % n, i = p / (n * n);
        cases[q] = (uint8_t)cell_case(f, n, iso, p, i, j, k);
        nt += g_mc_ntri[cases[q]];
        const uint32_t L = local[p], m = L >> LOCAL_BITS;
        uint64_t vi = base_v[blockIdx.x] + (L & ((1u << LOCAL_BITS) - 1u));
        const uint32_t stride[3] = {n * n, n, 1u};
#pragma unroll
        for (uint32_t a = 0; a < 3; ++a) {
            if (!((m >> a) & 1u)) continue;
            const float fa = f[p], fb = f[p + stride[a]];
            const float t = __fdiv_rn(iso - fa, fb - fa);
            float c[3] = {(float)i, (float)j, (float)k};
            c[a] = c[a] + t;
            verts[3 * vi] = __fdiv_rn(c[1], fn);
            verts[3 * vi + 1] = __fdiv_rn(c[0], fn);
            verts[3 * vi + 2] = __fdiv_rn(c[2], fn);
            ++vi;
        }
    }
    uint32_t tot;
    uint64_t ti = base_t[blockIdx.x] + block_excl_scan<uint32_t>(nt, sh, tot);   // (also orders the table staging before its reads)
#pragma unroll 1
    for (uint32_t q = 0; q < MC_PPT; ++q) {
        const uint32_t cs = cases[q];
        if (!cs) continue;
        const uint32_t p = p0 + q;
        for (uint32_t s = 0; s < 3 * NGP_MC_MAX_TRIS && s_tri[cs][s] >= 0; s += 3, ++ti) {
#pragma unroll
            for (uint32_t v = 0; v < 3; ++v) {
                const uint32_t e = (uint32_t)s_tri[cs][s + v], a = e >> 2, q4 = e & 3;
                // lowest corner of cube edge e: the q4-th corner (ascending) whose bit `a` is clear
                const uint32_t lo = a == 0 ? 2 * q4 : a == 1 ? (q4 & 1) | ((q4 & 2) << 1) : q4;
                const uint32_t pp = p + (lo & 1) * n * n + ((lo >> 1) & 1) * n + ((lo >> 2) & 1);
                tris[3 * ti + v] = (int32_t)edge_vertex(local, base_v, pp, a);
            }
        }
    }
}

// ---- u32 exclusive scan in place (a[0..len) -> prefix sums; *total = sum) --------------------------------
__global__ void __launch_bounds__(SC_THREADS) scan_part_kernel(const uint32_t* __restrict__ a, uint32_t len, uint32_t* __restrict__ bsum) {
    __shared__ uint32_t sh[32];
    const uint32_t i0 = blockIdx.x * SC_BLOCK + threadIdx.x * SC_PPT;
    uint32_t s = 0;
#pragma unroll
    for (uint32_t q = 0; q < SC_PPT; ++q)
        if (i0 + q < len) s += a[i0 + q];
    uint32_t tot;
    block_excl_scan<uint32_t>(s, sh, tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(TOP_THREADS) scan_top_kernel(uint32_t* __restrict__ bsum, uint32_t nb, uint32_t* __restrict__ total) {
    top_scan<uint32_t>(bsum, bsum, nb, total);
}
__global__ void __launch_bounds__(SC_THREADS) scan_apply_kernel(uint32_t* __restrict__ a, uint32_t len, const uint32_t* __restrict__ bsum) {
    __shared__ uint32_t sh[32];
    const uint32_t i0 = blockIdx.x * SC_BLOCK + threadIdx.x * SC_PPT;
    uint32_t v[SC_PPT], s = 0;
#pragma unroll
    for (uint32_t q = 0; q < SC_PPT; ++q) { v[q] = i0 + q < len ? a[i0 + q] : 0u; s += v[q]; }
    uint32_t tot;
    uint32_t run = bsum[blockIdx.x] + block_excl_scan<uint32_t>(s, sh, tot);
#pragma unroll
    for (uint32_t q = 0; q < SC_PPT; ++q)
        if (i0 + q < len) { a[i0 + q] = run; run += v[q]; }
}

// ---- vertex -> triangle incidence (CSR), shared by the component filter and the normals --------------------
__global__ void deg_kernel(uint32_t nv, uint32_t nt, const int32_t* __restrict__ tris, uint32_t* __restrict__ deg, uint32_t* __restrict__ status) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
#pragma unroll
    for (uint32_t c = 0; c < 3; ++c) {
        const uint32_t v = (uint32_t)tris[3 * (size_t)t + c];
        if (v < nv) atomicAdd(deg + v, 1u);
        else atomicOr(status, 1u);
    }
}
__global__ void fill_kernel(uint32_t nv, uint32_t nt, const int32_t* __restrict__ tris, const uint32_t* __restrict__ off, uint32_t* __restrict__ cur,
                            uint32_t* __restrict__ inc) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
#pragma unroll
    for (uint32_t c = 0; c < 3; ++c) {
        const uint32_t v = (uint32_t)tris[3 * (size_t)t + c];
        if (v < nv) inc[off[v] + atomicAdd(cur + v, 1u)] = t;
    }
}
// the incidence lists were filled in arbitrary order: sort each ascending, so that everything read from them is deterministic
__global__ void sort_kernel(uint32_t nv, const uint32_t* __restrict__ off, uint32_t* __restrict__ inc) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const uint32_t lo = off[v], hi = off[v + 1];
    for (uint32_t i = lo + 1; i < hi; ++i) {
        const uint32_t x = inc[i];
        uint32_t j = i;
        for (; j > lo && inc[j - 1] > x; --j) inc[j] = inc[j - 1];
        inc[j] = x;
    }
}

// ---- largest component ----------------------------------------------------------------------------------
// Union-find with the smaller root as the new root: a root is always the smallest triangle of its set, whatever the order of the
// unions.  find() halves paths with plain stores: every store points a node at one of its ancestors, so a lost store costs nothing.
__device__ __forceinline__ uint32_t uf_find(volatile uint32_t* p, uint32_t x) {
    uint32_t y = p[x];
    while (y != x) {
        const uint32_t z = p[y];
        if (z != y) p[x] = z;
        x = y;
        y = z;
    }
    return x;
}
__device__ __forceinline__ void uf_union(uint32_t* p, uint32_t a, uint32_t b) {
    volatile uint32_t* vp = p;
    while (true) {
        a = uf_find(vp, a);
        b = uf_find(vp, b);
        if (a == b) return;
        if (a > b) { const uint32_t s = a; a = b; b = s; }
        const uint32_t old = atomicCAS(p + b, b, a);                    // hook the larger root under the smaller one
        if (old == b) return;
        b = old;
    }
}
__device__ __forceinline__ uint64_t edge_key(uint32_t a, uint32_t b) { return a < b ? ((uint64_t)a << 32 | b) : ((uint64_t)b << 32 | a); }

__global__ void init_parent_kernel(uint32_t nt, uint32_t* __restrict__ parent) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < nt) parent[t] = t;
}
// joins triangle t with every later triangle that shares one of its edges (as an unordered vertex pair, like Open3D)
__global__ void union_kernel(uint32_t nv, uint32_t nt, const int32_t* __restrict__ tris, const uint32_t* __restrict__ off, const uint32_t* __restrict__ inc,
                             uint32_t* parent) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    uint32_t tv[3];
#pragma unroll
    for (uint32_t c = 0; c < 3; ++c) tv[c] = (uint32_t)tris[3 * (size_t)t + c];
#pragma unroll 1
    for (uint32_t c = 0; c < 3; ++c) {
        const uint32_t a = tv[c], b = tv[(c + 1) % 3];
        if (a >= nv || b >= nv) continue;
        const uint64_t key = edge_key(a, b);
        for (uint32_t i = off[a]; i < off[a + 1]; ++i) {
            const uint32_t s = inc[i];
            if (s <= t) continue;
            const uint32_t s0 = (uint32_t)tris[3 * (size_t)s], s1 = (uint32_t)tris[3 * (size_t)s + 1], s2 = (uint32_t)tris[3 * (size_t)s + 2];
            if (edge_key(s0, s1) == key || edge_key(s1, s2) == key || edge_key(s2, s0) == key) uf_union(parent, t, s);
        }
    }
}
// final labels (each triangle -> its root) and the cluster sizes
__global__ void label_count_kernel(uint32_t nt, uint32_t* parent, uint32_t* __restrict__ cnt) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const uint32_t r = uf_find(parent, t);
    atomicAdd(cnt + r, 1u);
}
// the largest cluster, on a tie the one with the smallest label: max of (count, ~label)
__global__ void best_kernel(uint32_t nt, const uint32_t* __restrict__ cnt, unsigned long long* __restrict__ best) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < nt && cnt[t]) atomicMax(best, (unsigned long long)cnt[t] << 32 | (0xffffffffu - t));
}
__device__ __forceinline__ uint32_t best_label(const unsigned long long* best) { return 0xffffffffu - (uint32_t)(*best & 0xffffffffu); }
// keep flags of the triangles, use flags of their vertices
__global__ void keep_kernel(uint32_t nv, uint32_t nt, const int32_t* __restrict__ tris, uint32_t* parent, const unsigned long long* __restrict__ best,
                            uint32_t* __restrict__ keep_t, uint32_t* __restrict__ use_v) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const bool k = uf_find(parent, t) == best_label(best);
    keep_t[t] = k;
    if (k)
#pragma unroll
        for (uint32_t c = 0; c < 3; ++c) {
            const uint32_t v = (uint32_t)tris[3 * (size_t)t + c];
            if (v < nv) use_v[v] = 1u;
        }
}
// order-preserving compaction (keep_t / use_v now hold their exclusive prefix sums; totals[0..1] = kept vertices, triangles)
__global__ void compact_kernel(uint32_t nv, uint32_t nt, const float* __restrict__ verts, const int32_t* __restrict__ tris, const uint32_t* __restrict__ new_t,
                               const uint32_t* __restrict__ new_v, const uint32_t* __restrict__ totals, float* __restrict__ verts_out,
                               int32_t* __restrict__ tris_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nv && (i + 1 < nv ? new_v[i + 1] : totals[0]) != new_v[i]) {
#pragma unroll
        for (uint32_t c = 0; c < 3; ++c) verts_out[3 * (size_t)new_v[i] + c] = verts[3 * (size_t)i + c];
    }
    if (i < nt && (i + 1 < nt ? new_t[i + 1] : totals[1]) != new_t[i]) {
#pragma unroll
        for (uint32_t c = 0; c < 3; ++c) {
            const uint32_t v = (uint32_t)tris[3 * (size_t)i + c];
            tris_out[3 * (size_t)new_t[i] + c] = v < nv ? (int32_t)new_v[v] : -1;
        }
    }
}

// ---- normals ------------------------------------------------------------------------------------------
// each vertex sums the unnormalised cross products of its triangles in ascending triangle order (a fixed-order gather), then normalises
__global__ void normals_kernel(uint32_t nv, const float* __restrict__ verts, const int32_t* __restrict__ tris, const uint32_t* __restrict__ off,
                               const uint32_t* __restrict__ inc, float* __restrict__ normals) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (uint32_t i = off[v]; i < off[v + 1]; ++i) {
        const size_t s = inc[i];
        const float* p0 = verts + 3 * (size_t)(uint32_t)tris[3 * s];
        const float* p1 = verts + 3 * (size_t)(uint32_t)tris[3 * s + 1];
        const float* p2 = verts + 3 * (size_t)(uint32_t)tris[3 * s + 2];
        const float ux = p1[0] - p0[0], uy = p1[1] - p0[1], uz = p1[2] - p0[2];
        const float vx = p2[0] - p0[0], vy = p2[1] - p0[1], vz = p2[2] - p0[2];
        nx = nx + (uy * vz - uz * vy);
        ny = ny + (uz * vx - ux * vz);
        nz = nz + (ux * vy - uy * vx);
    }
    const float len = __fsqrt_rn(nx * nx + ny * ny + nz * nz);
    if (len > 0.f) { nx = __fdiv_rn(nx, len); ny = __fdiv_rn(ny, len); nz = __fdiv_rn(nz, len); }
    normals[3 * (size_t)v] = nx;
    normals[3 * (size_t)v + 1] = ny;
    normals[3 * (size_t)v + 2] = nz;
}

// ---- workspace layouts ------------------------------------------------------------------------------------
inline uint64_t al(uint64_t b) { return (b + 255) & ~uint64_t(255); }
struct McWs {
    uint16_t* local; uint32_t *bcnt_v, *bcnt_t; uint64_t *base_v, *base_t, *totals;
    static uint64_t layout(uint32_t n, uint8_t* w, McWs* o) {
        const uint64_t n3 = (uint64_t)n * n * n, nb = (n3 + MC_BLOCK - 1) / MC_BLOCK;
        uint64_t at = 0;
        auto take = [&](uint64_t bytes) { uint8_t* p = w ? w + at : nullptr; at += al(bytes); return p; };
        uint8_t* l = take(2 * n3); uint8_t* cv = take(4 * nb); uint8_t* ct = take(4 * nb);
        uint8_t* bv = take(8 * nb); uint8_t* bt = take(8 * nb); uint8_t* tt = take(16);
        if (o) *o = McWs{(uint16_t*)l, (uint32_t*)cv, (uint32_t*)ct, (uint64_t*)bv, (uint64_t*)bt, (uint64_t*)tt};
        return at;
    }
};
struct MeshWs {
    uint32_t *off, *cur, *inc, *parent, *cnt, *new_t, *new_v, *bsum, *small;   // small: status, totals[2], pad
    unsigned long long* best;
    static uint64_t layout(uint64_t nv, uint64_t nt, uint8_t* w, MeshWs* o) {
        const uint64_t len = nv + 1 > nt ? nv + 1 : nt, nb = (len + SC_BLOCK - 1) / SC_BLOCK;
        uint64_t at = 0;
        auto take = [&](uint64_t bytes) { uint8_t* p = w ? w + at : nullptr; at += al(bytes); return p; };
        uint8_t* off = take(4 * (nv + 1)); uint8_t* cur = take(4 * nv); uint8_t* inc = take(12 * nt); uint8_t* par = take(4 * nt);
        uint8_t* cnt = take(4 * nt); uint8_t* nt_ = take(4 * nt); uint8_t* nv_ = take(4 * nv); uint8_t* bs = take(4 * nb);
        uint8_t* sm = take(16); uint8_t* be = take(8);
        if (o) *o = MeshWs{(uint32_t*)off, (uint32_t*)cur, (uint32_t*)inc, (uint32_t*)par, (uint32_t*)cnt, (uint32_t*)nt_, (uint32_t*)nv_, (uint32_t*)bs,
                           (uint32_t*)sm, (unsigned long long*)be};
        return at;
    }
};

inline uint32_t blocks(uint64_t n, uint32_t per) { return (uint32_t)((n + per - 1) / per); }

}  // namespace

// exclusive scan of a[0..len) in place, sum -> *total (device)
int ngp_mesh::scan_u32(cudaStream_t s, uint32_t* a, uint32_t len, uint32_t* bsum, uint32_t* total) {
    const uint32_t nb = blocks(len, SC_BLOCK);
    if (nb == 0) return 0;
    scan_part_kernel<<<nb, SC_THREADS, 0, s>>>(a, len, bsum);
    NGP_LAUNCH_CHECK();
    scan_top_kernel<<<1, TOP_THREADS, 0, s>>>(bsum, nb, total);
    NGP_LAUNCH_CHECK();
    scan_apply_kernel<<<nb, SC_THREADS, 0, s>>>(a, len, bsum);
    NGP_LAUNCH_CHECK();
    return 0;
}

namespace {

// vertex -> triangle incidence lists, each ascending; status bit 0 = a triangle index out of range (that corner is ignored)
int build_csr(cudaStream_t s, uint32_t nv, uint32_t nt, const int32_t* tris, const MeshWs& w) {
    NGP_CHECK_CUDA(cudaMemsetAsync(w.off, 0, 4 * ((size_t)nv + 1), s));
    NGP_CHECK_CUDA(cudaMemsetAsync(w.cur, 0, 4 * (size_t)nv, s));
    NGP_CHECK_CUDA(cudaMemsetAsync(w.small, 0, 16, s));
    deg_kernel<<<blocks(nt, 256), 256, 0, s>>>(nv, nt, tris, w.off, w.small);
    NGP_LAUNCH_CHECK();
    if (int rc = scan_u32(s, w.off, nv, w.bsum, w.off + nv)) return rc;
    fill_kernel<<<blocks(nt, 256), 256, 0, s>>>(nv, nt, tris, w.off, w.cur, w.inc);
    NGP_LAUNCH_CHECK();
    sort_kernel<<<blocks(nv, 256), 256, 0, s>>>(nv, w.off, w.inc);
    NGP_LAUNCH_CHECK();
    return 0;
}

int check_mesh_sizes(const char* fn, uint64_t nv, uint64_t nt) {
    NGP_REQUIRE(nv <= 0x7fffffffull && nt <= 0x7fffffffull,
                std::string(fn) + ": at most 2^31 - 1 vertices and triangles (indices are int32), got " + std::to_string(nv) + " / " + std::to_string(nt));
    return 0;
}

}  // namespace

extern "C" {

int ngp_mesh_workspace_bytes(uint32_t n, uint64_t n_verts, uint64_t n_tris, uint64_t* bytes_out) {
    NGP_REQUIRE(n == 0 || (n >= 2 && n <= 1024), "ngp_mesh_workspace_bytes: resolution n must be 0 or in [2, 1024], got " + std::to_string(n));
    if (int rc = check_mesh_sizes("ngp_mesh_workspace_bytes", n_verts, n_tris)) return rc;
    NGP_REQUIRE(bytes_out, "ngp_mesh_workspace_bytes: bytes_out is required");
    const uint64_t a = n ? McWs::layout(n, nullptr, nullptr) : 0, b = MeshWs::layout(n_verts, n_tris, nullptr, nullptr);
    *bytes_out = a > b ? a : b;
    return 0;
}

int ngp_marching_cubes(void* stream, uint32_t n, const float* field, float iso, void* workspace, float* verts, uint64_t max_verts, int32_t* tris,
                       uint64_t max_tris, uint64_t* counts_host) {
    NGP_REQUIRE(n >= 2 && n <= 1024, "ngp_marching_cubes: resolution n must be in [2, 1024], got " + std::to_string(n));
    NGP_REQUIRE(field && workspace && counts_host, "ngp_marching_cubes: field, workspace and counts_host are required");
    cudaStream_t s = (cudaStream_t)stream;
    McWs w;
    McWs::layout(n, (uint8_t*)workspace, &w);
    const uint32_t n3 = n * n * n, nb = blocks(n3, MC_BLOCK);
    mc_count_kernel<<<nb, MC_THREADS, 0, s>>>(n, field, iso, w.local, w.bcnt_v, w.bcnt_t);
    NGP_LAUNCH_CHECK();
    mc_scan_kernel<<<1, TOP_THREADS, 0, s>>>(w.bcnt_v, w.bcnt_t, w.base_v, w.base_t, nb, w.totals);
    NGP_LAUNCH_CHECK();
    uint64_t tot[2];
    NGP_CHECK_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    counts_host[0] = tot[0];
    counts_host[1] = tot[1];
    if (!verts && !tris) return 0;                                       // count only
    NGP_REQUIRE(verts && tris, "ngp_marching_cubes: pass both output buffers, or neither to count");
    NGP_REQUIRE(tot[0] <= max_verts && tot[1] <= max_tris, "ngp_marching_cubes: output capacity " + std::to_string(max_verts) + " vertices / " +
                std::to_string(max_tris) + " triangles, the mesh has " + std::to_string(tot[0]) + " / " + std::to_string(tot[1]));
    if (int rc = check_mesh_sizes("ngp_marching_cubes", tot[0], tot[1])) return rc;
    mc_emit_kernel<<<nb, MC_THREADS, 0, s>>>(n, field, iso, w.local, w.base_v, w.base_t, verts, tris);
    NGP_LAUNCH_CHECK();
    return 0;
}

int ngp_mesh_largest_component(void* stream, uint64_t n_verts, uint64_t n_tris, const float* verts, const int32_t* tris, void* workspace,
                               float* verts_out, int32_t* tris_out, uint64_t* counts_host) {
    if (int rc = check_mesh_sizes("ngp_mesh_largest_component", n_verts, n_tris)) return rc;
    NGP_REQUIRE(counts_host, "ngp_mesh_largest_component: counts_host is required");
    counts_host[0] = counts_host[1] = 0;
    if (n_tris == 0) return 0;
    NGP_REQUIRE(verts && tris && workspace && verts_out && tris_out, "ngp_mesh_largest_component: null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nv = (uint32_t)n_verts, nt = (uint32_t)n_tris;
    MeshWs w;
    MeshWs::layout(nv, nt, (uint8_t*)workspace, &w);
    if (int rc = build_csr(s, nv, nt, tris, w)) return rc;
    init_parent_kernel<<<blocks(nt, 256), 256, 0, s>>>(nt, w.parent);
    NGP_LAUNCH_CHECK();
    union_kernel<<<blocks(nt, 256), 256, 0, s>>>(nv, nt, tris, w.off, w.inc, w.parent);
    NGP_LAUNCH_CHECK();
    NGP_CHECK_CUDA(cudaMemsetAsync(w.cnt, 0, 4 * (size_t)nt, s));
    NGP_CHECK_CUDA(cudaMemsetAsync(w.new_v, 0, 4 * (size_t)nv, s));
    NGP_CHECK_CUDA(cudaMemsetAsync(w.best, 0, 8, s));
    label_count_kernel<<<blocks(nt, 256), 256, 0, s>>>(nt, w.parent, w.cnt);
    NGP_LAUNCH_CHECK();
    best_kernel<<<blocks(nt, 256), 256, 0, s>>>(nt, w.cnt, w.best);
    NGP_LAUNCH_CHECK();
    keep_kernel<<<blocks(nt, 256), 256, 0, s>>>(nv, nt, tris, w.parent, w.best, w.new_t, w.new_v);
    NGP_LAUNCH_CHECK();
    if (int rc = scan_u32(s, w.new_v, nv, w.bsum, w.small + 1)) return rc;
    if (int rc = scan_u32(s, w.new_t, nt, w.bsum, w.small + 2)) return rc;
    const uint32_t nmax = nv > nt ? nv : nt;
    compact_kernel<<<blocks(nmax, 256), 256, 0, s>>>(nv, nt, verts, tris, w.new_t, w.new_v, w.small + 1, verts_out, tris_out);
    NGP_LAUNCH_CHECK();
    uint32_t sm[3];
    NGP_CHECK_CUDA(cudaMemcpyAsync(sm, w.small, sizeof(sm), cudaMemcpyDeviceToHost, s));
    NGP_CHECK_CUDA(cudaStreamSynchronize(s));
    NGP_REQUIRE(!(sm[0] & 1u), "ngp_mesh_largest_component: a triangle index is outside [0, n_verts)");
    counts_host[0] = sm[1];
    counts_host[1] = sm[2];
    return 0;
}

int ngp_mesh_vertex_normals(void* stream, uint64_t n_verts, uint64_t n_tris, const float* verts, const int32_t* tris, void* workspace, float* normals) {
    if (int rc = check_mesh_sizes("ngp_mesh_vertex_normals", n_verts, n_tris)) return rc;
    if (n_verts == 0) return 0;
    NGP_REQUIRE(verts && normals && workspace && (tris || n_tris == 0), "ngp_mesh_vertex_normals: null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nv = (uint32_t)n_verts, nt = (uint32_t)n_tris;
    MeshWs w;
    MeshWs::layout(nv, nt, (uint8_t*)workspace, &w);
    if (int rc = build_csr(s, nv, nt, tris, w)) return rc;
    normals_kernel<<<blocks(nv, 256), 256, 0, s>>>(nv, verts, tris, w.off, w.inc, normals);
    NGP_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
