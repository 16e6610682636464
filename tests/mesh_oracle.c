/*
 * mesh_oracle.c -- CPU restatement of mesh extraction (tools/extract_mesh.py of the JNeRF reference).  TEST INFRASTRUCTURE ONLY:
 * compiled on first use by tests/mesh_oracle.py (gcc, -ffp-contract=off) and loaded by tests/ and tools/gen_mc_table.py; the product
 * (libngp_b200.so) never links, includes or calls it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------------
 * Mesh extraction (tools/extract_mesh.py:42-106).  The reference hands the work to PyMCubes
 * (marching_cubes, :78), Open3D (cluster_connected_triangles + remove_unreferenced_vertices, :92-97;
 * compute_vertex_normals, :106) and writes PLY files with plyfile; none of those packages is restated
 * bit for bit (their vertex order cannot be checked without them).  What is restated is the behaviour
 * fixed in DESIGN.md section 7 "Mesh extraction".
 *
 * Lattice: field index (i*N + j)*N + k.  Cube corner c = (c&1, c>>1&1, c>>2&1) along (i, j, k); cube edge
 * e = 4*axis + q joins the q-th corner (ascending) whose `axis` bit is clear to its neighbour along `axis`.
 * A corner is inside when f > iso.  Lattice edge (p, axis) crosses when exactly one endpoint is inside.
 * ---------------------------------------------------------------------------------------------- */
#define ORC_MC_MAXT 5
static int mc_edge_lo(int e) {
    int a = e >> 2, q = e & 3, n = 0;
    for (int c = 0; c < 8; ++c)
        if (!((c >> a) & 1)) { if (n == q) return c; ++n; }
    return -1;
}
static int mc_edge_of(int c0, int c1) {
    int lo = c0 < c1 ? c0 : c1, a = (c0 ^ c1) == 1 ? 0 : (c0 ^ c1) == 2 ? 1 : 2;
    for (int q = 0; q < 4; ++q)
        if (mc_edge_lo(4 * a + q) == lo) return 4 * a + q;
    return -1;
}
static void mc_corner_pos(int c, float* p) { p[0] = (float)(c & 1); p[1] = (float)((c >> 1) & 1); p[2] = (float)((c >> 2) & 1); }
static void mc_edge_mid(int e, float* p) { mc_corner_pos(mc_edge_lo(e), p); p[e >> 2] += 0.5f; }

/* two cube edges lie on one face when they are parallel neighbours on it or meet at a corner */
static int mc_share_face(int e0, int e1) {
    const int a0 = e0 >> 2, a1 = e1 >> 2, c0 = mc_edge_lo(e0), c1 = mc_edge_lo(e1);
    for (int a = 0; a < 3; ++a) {                                         /* face: bit a of every corner = side */
        if (a == a0 || a == a1) continue;
        if (((c0 >> a) & 1) == ((c1 >> a) & 1)) return 1;
    }
    return 0;
}
static int g_mc_bad = 0;
static int8_t g_mc_tri[256][3 * ORC_MC_MAXT];
static uint8_t g_mc_ntri[256];
static int g_mc_ready = 0;

/* The 256-case table from its rule.  On every cube face, each run of inside corners is cut off by one segment between the two
 * crossing edges that bound the run (an ambiguous face -- two diagonal inside corners -- gets two segments: the inside corners are
 * separated).  The rule depends on the face's four corners only, so the two cubes sharing a face cut it alike: no cracks.  Each
 * segment is directed so that, seen from outside the cube, the inside corners lie to its right; the segments then chain into closed
 * cycles, one per surface piece, taken in order of their lowest edge and walked from it.  Cycle (c0 c1 .. c_{m-1}) becomes the fan
 * (c_r, c_{r+s+1}, c_{r+s}), s = 1 .. m-2, from the first root r that draws no diagonal between two edges of one face: in the lattice frame (i, j, k) the triangles face the inside; the x/y swap of the PLY frame is a
 * mirror, so there they face the outside (towards lower density). */
static void mc_build_table(void) {
    if (g_mc_ready) return;
    for (int m = 0; m < 256; ++m) {
        int next[12];
        for (int e = 0; e < 12; ++e) next[e] = -1;
        for (int a = 0; a < 3; ++a)
            for (int s = 0; s < 2; ++s) {
                static const int ub[4] = {0, 1, 1, 0}, ud[4] = {0, 0, 1, 1};
                int b = (a + 1) % 3, d = (a + 2) % 3, cyc[4];
                for (int q = 0; q < 4; ++q) cyc[q] = (s << a) | (ub[q] << b) | (ud[q] << d);
                for (int q = 0; q < 4; ++q) {
                    if (((m >> cyc[q]) & 1) || !((m >> cyc[(q + 1) & 3]) & 1)) continue;   /* run of inside corners starts at q+1 */
                    int r = (q + 1) & 3;
                    while ((m >> cyc[(r + 1) & 3]) & 1) r = (r + 1) & 3;                  /* ... and ends at r */
                    int e0 = mc_edge_of(cyc[q], cyc[(q + 1) & 3]), e1 = mc_edge_of(cyc[r], cyc[(r + 1) & 3]);
                    float P[3], Q[3], C[3], u[3], v[3], x[3], nrm[3] = {0, 0, 0};
                    mc_edge_mid(e0, P); mc_edge_mid(e1, Q); mc_corner_pos(cyc[(q + 1) & 3], C);
                    nrm[a] = s ? 1.f : -1.f;
                    for (int k = 0; k < 3; ++k) { u[k] = Q[k] - P[k]; v[k] = C[k] - P[k]; }
                    x[0] = u[1] * v[2] - u[2] * v[1]; x[1] = u[2] * v[0] - u[0] * v[2]; x[2] = u[0] * v[1] - u[1] * v[0];
                    if (x[0] * nrm[0] + x[1] * nrm[1] + x[2] * nrm[2] < 0) next[e0] = e1; else next[e1] = e0;
                }
            }
        int seen[12] = {0}, nt = 0;
        for (int e = 0; e < 12; ++e) {
            if (next[e] < 0 || seen[e]) continue;
            int cyc[12], len = 0, x = e;
            do { seen[x] = 1; cyc[len++] = x; x = next[x]; } while (x != e && x >= 0 && len < 12);
            /* fan root: the first cycle vertex none of whose diagonals joins two edges of one cube face.  Such a diagonal can only cross
             * an ambiguous face, and the cube on its other side might draw it too: the edge would then carry four triangles. */
            int root = -1;
            for (int r0 = 0; r0 < len && root < 0; ++r0) {
                int ok = 1;
                for (int s = 2; s + 1 < len; ++s) ok &= !mc_share_face(cyc[r0], cyc[(r0 + s) % len]);
                if (ok) root = r0;
            }
            if (root < 0) g_mc_bad = 1;
            if (root < 0) root = 0;
            for (int s = 1; s + 1 < len; ++s) {
                g_mc_tri[m][3 * nt] = (int8_t)cyc[root];
                g_mc_tri[m][3 * nt + 1] = (int8_t)cyc[(root + s + 1) % len];
                g_mc_tri[m][3 * nt + 2] = (int8_t)cyc[(root + s) % len];
                ++nt;
            }
        }
        for (int k = 3 * nt; k < 3 * ORC_MC_MAXT; ++k) g_mc_tri[m][k] = -1;
        g_mc_ntri[m] = (uint8_t)nt;
    }
    g_mc_ready = 1;
}
/* the table (256 x 3*ORC_MC_MAXT cube-edge ids, -1 padded) and the triangle count of every case; returns ORC_MC_MAXT, or -1 when a
 * cycle had no admissible fan root */
int orc_mc_table(int8_t* tri, uint8_t* ntri) {
    mc_build_table();
    if (g_mc_bad) return -1;
    memcpy(tri, g_mc_tri, sizeof(g_mc_tri));
    memcpy(ntri, g_mc_ntri, sizeof(g_mc_ntri));
    return ORC_MC_MAXT;
}

static inline int mc_in(float v, float iso) { return v > iso; }
static inline unsigned mc_mask(uint32_t n, const float* f, float iso, uint32_t i, uint32_t j, uint32_t k) {
    const uint64_t p = ((uint64_t)i * n + j) * n + k;
    const int a = mc_in(f[p], iso);
    unsigned m = 0;
    if (i + 1 < n && a != mc_in(f[p + (uint64_t)n * n], iso)) m |= 1u;
    if (j + 1 < n && a != mc_in(f[p + n], iso)) m |= 2u;
    if (k + 1 < n && a != mc_in(f[p + 1], iso)) m |= 4u;
    return m;
}

/* PyMCubes' marching_cubes(sigma, iso) (:78) + the frame of :80-84 (vertex = lattice position / N, first two columns swapped).
 * Vertices in lattice-edge order (point index major, axis minor), each interpolated from the edge's lower endpoint a:
 * a + (iso - f_a) / (f_b - f_a).  Triangles in cell order, within a cell in table order.  counts[0..1] = vertices, triangles;
 * verts (V,3) / tris (T,3) may be NULL (count only).  Returns 0, or 1 when a count exceeds its capacity (nothing past it written). */
int orc_marching_cubes(uint32_t n, const float* f, float iso, float* verts, int32_t* tris, uint64_t max_v, uint64_t max_t, uint64_t* counts) {
    mc_build_table();
    const uint64_t n3 = (uint64_t)n * n * n, s[3] = {(uint64_t)n * n, n, 1};
    uint32_t* pre = (uint32_t*)malloc(sizeof(uint32_t) * (n3 ? n3 : 1));     /* vertices on the points before p */
    uint64_t nv = 0, nt = 0;
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = 0; j < n; ++j)
            for (uint32_t k = 0; k < n; ++k) {
                const uint64_t p = ((uint64_t)i * n + j) * n + k;
                pre[p] = (uint32_t)nv;
                const unsigned m = mc_mask(n, f, iso, i, j, k);
                for (int a = 0; a < 3; ++a) {
                    if (!((m >> a) & 1)) continue;
                    if (verts && nv < max_v) {
                        const float fa = f[p], fb = f[p + s[a]];
                        const float t = (iso - fa) / (fb - fa);
                        float c[3] = {(float)i, (float)j, (float)k};
                        c[a] = c[a] + t;
                        verts[3 * nv] = c[1] / (float)n; verts[3 * nv + 1] = c[0] / (float)n; verts[3 * nv + 2] = c[2] / (float)n;
                    }
                    ++nv;
                }
            }
    for (uint32_t i = 0; i + 1 < n; ++i)
        for (uint32_t j = 0; j + 1 < n; ++j)
            for (uint32_t k = 0; k + 1 < n; ++k) {
                const uint64_t p = ((uint64_t)i * n + j) * n + k;
                unsigned cs = 0;
                for (int c = 0; c < 8; ++c)
                    cs |= (unsigned)mc_in(f[p + (c & 1) * s[0] + ((c >> 1) & 1) * s[1] + ((c >> 2) & 1) * s[2]], iso) << c;
                for (int q = 0; q < g_mc_ntri[cs]; ++q, ++nt) {
                    if (!tris || nt >= max_t) continue;
                    for (int v = 0; v < 3; ++v) {
                        const int e = g_mc_tri[cs][3 * q + v], lo = mc_edge_lo(e), a = e >> 2;
                        const uint32_t ci = i + (lo & 1), cj = j + ((lo >> 1) & 1), ck = k + ((lo >> 2) & 1);
                        const uint64_t pp = ((uint64_t)ci * n + cj) * n + ck;
                        const unsigned mm = mc_mask(n, f, iso, ci, cj, ck);
                        tris[3 * nt + v] = (int32_t)(pre[pp] + (uint32_t)__builtin_popcount(mm & ((1u << a) - 1u)));
                    }
                }
            }
    free(pre);
    counts[0] = nv;
    counts[1] = nt;
    return (verts && nv > max_v) || (tris && nt > max_t);
}

typedef struct { uint64_t key; uint32_t tri; } orc_edge_rec;
static int orc_edge_cmp(const void* a, const void* b) {
    const uint64_t x = ((const orc_edge_rec*)a)->key, y = ((const orc_edge_rec*)b)->key;
    return x < y ? -1 : x > y;
}
/* Open3D's cluster_connected_triangles + argmax + remove_triangles_by_index + remove_unreferenced_vertices (:92-97): triangles are
 * in one cluster when a chain of shared edges joins them; clusters are found by breadth-first search from the lowest unvisited
 * triangle, so cluster ids grow with their lowest triangle and np.argmax keeps, on a tie, the cluster of the lowest triangle.
 * Kept triangles and vertices keep their order; indices are remapped.  counts[0..1] = kept vertices, kept triangles. */
void orc_mesh_largest_component(uint64_t nv, uint64_t nt, const float* verts, const int32_t* tris, float* verts_out, int32_t* tris_out,
                                uint64_t* counts) {
    counts[0] = counts[1] = 0;
    if (!nt) return;
    orc_edge_rec* ed = (orc_edge_rec*)malloc(sizeof(orc_edge_rec) * 3 * nt);
    for (uint64_t t = 0; t < nt; ++t)
        for (int c = 0; c < 3; ++c) {
            uint64_t a = (uint32_t)tris[3 * t + c], b = (uint32_t)tris[3 * t + (c + 1) % 3];
            ed[3 * t + c].key = a < b ? (a << 32 | b) : (b << 32 | a);
            ed[3 * t + c].tri = (uint32_t)t;
        }
    qsort(ed, 3 * nt, sizeof(orc_edge_rec), orc_edge_cmp);
    int64_t* cl = (int64_t*)malloc(sizeof(int64_t) * nt);
    uint32_t* queue = (uint32_t*)malloc(sizeof(uint32_t) * nt);
    uint64_t* cnt = (uint64_t*)calloc(nt, sizeof(uint64_t));
    for (uint64_t t = 0; t < nt; ++t) cl[t] = -1;
    int64_t ncl = 0;
    for (uint64_t t0 = 0; t0 < nt; ++t0) {
        if (cl[t0] >= 0) continue;
        uint64_t head = 0, tail = 0;
        queue[tail++] = (uint32_t)t0;
        cl[t0] = ncl;
        while (head < tail) {
            const uint32_t t = queue[head++];
            ++cnt[ncl];
            for (int c = 0; c < 3; ++c) {
                uint64_t a = (uint32_t)tris[3 * (uint64_t)t + c], b = (uint32_t)tris[3 * (uint64_t)t + (c + 1) % 3];
                const uint64_t key = a < b ? (a << 32 | b) : (b << 32 | a);
                uint64_t lo = 0, hi = 3 * nt;                                     /* first record with this edge */
                while (lo < hi) { uint64_t mid = (lo + hi) / 2; if (ed[mid].key < key) lo = mid + 1; else hi = mid; }
                for (; lo < 3 * nt && ed[lo].key == key; ++lo)
                    if (cl[ed[lo].tri] < 0) { cl[ed[lo].tri] = ncl; queue[tail++] = ed[lo].tri; }
            }
        }
        ++ncl;
    }
    int64_t best = 0;
    for (int64_t c = 1; c < ncl; ++c)
        if (cnt[c] > cnt[best]) best = c;
    int64_t* remap = (int64_t*)malloc(sizeof(int64_t) * (nv ? nv : 1));
    for (uint64_t v = 0; v < nv; ++v) remap[v] = -1;
    for (uint64_t t = 0; t < nt; ++t)
        if (cl[t] == best)
            for (int c = 0; c < 3; ++c) remap[tris[3 * t + c]] = 0;
    uint64_t kv = 0, kt = 0;
    for (uint64_t v = 0; v < nv; ++v)
        if (remap[v] >= 0) {
            remap[v] = (int64_t)kv;
            memcpy(verts_out + 3 * kv, verts + 3 * v, 3 * sizeof(float));
            ++kv;
        }
    for (uint64_t t = 0; t < nt; ++t)
        if (cl[t] == best) {
            for (int c = 0; c < 3; ++c) tris_out[3 * kt + c] = (int32_t)remap[tris[3 * t + c]];
            ++kt;
        }
    counts[0] = kv;
    counts[1] = kt;
    free(ed); free(cl); free(queue); free(cnt); free(remap);
}

/* Open3D's compute_vertex_normals (:106): every vertex sums the unnormalised cross products (v1 - v0) x (v2 - v0) of its triangles,
 * in triangle order, then the sum is divided by its length (a zero sum stays zero).  fp32, no contraction. */
void orc_mesh_vertex_normals(uint64_t nv, uint64_t nt, const float* verts, const int32_t* tris, float* normals) {
    memset(normals, 0, sizeof(float) * 3 * nv);
    for (uint64_t t = 0; t < nt; ++t) {
        const float* p0 = verts + 3 * (uint64_t)tris[3 * t];
        const float* p1 = verts + 3 * (uint64_t)tris[3 * t + 1];
        const float* p2 = verts + 3 * (uint64_t)tris[3 * t + 2];
        const float ux = p1[0] - p0[0], uy = p1[1] - p0[1], uz = p1[2] - p0[2];
        const float vx = p2[0] - p0[0], vy = p2[1] - p0[1], vz = p2[2] - p0[2];
        const float cx = uy * vz - uz * vy, cy = uz * vx - ux * vz, cz = ux * vy - uy * vx;
        for (int c = 0; c < 3; ++c) {
            float* nn = normals + 3 * (uint64_t)tris[3 * t + c];
            nn[0] = nn[0] + cx; nn[1] = nn[1] + cy; nn[2] = nn[2] + cz;
        }
    }
    for (uint64_t v = 0; v < nv; ++v) {
        float* nn = normals + 3 * v;
        const float len = sqrtf(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]);
        if (len > 0.f) { nn[0] = nn[0] / len; nn[1] = nn[1] / len; nn[2] = nn[2] / len; }
    }
}
