// oracle/_ref build: the reference's Plenoxels sparse TV kernel (contrib/plenoxel loss_kernel.h) compiled UNMODIFIED for sm_90a, in
// its own translation unit (it redefines constants of volume_render_cuvol_fused.h), with tv_grad_sparse.py's launch shape.
// TEST / BENCH INFRASTRUCTURE: never linked into libngp_b200.so.
#include "loss_kernel.h"

// cells rand_cells (n,) of links (X, Y, Z); data (cap, dim); columns [0, dim); scale = lambda / n; grad (cap, dim) added to.
extern "C" int ref_svox_tv(int n, const int32_t* rand_cells, const int32_t* links, int X, int Y, int Z, const float* data, int cap, int dim,
                           float scale, int ignore_edge, float* grad, void* stream) {
    jittor::Var l{const_cast<int32_t*>(links), {X, Y, Z, 1}, (int64_t)X * Y * Z}, dv{const_cast<float*>(data), {cap, dim, 1, 1}, (int64_t)cap * dim};
    const size_t Q = (size_t)n * dim;
    tv_grad_sparse_kernel<<<CUDA_N_BLOCKS_NEEDED(Q, TV_GRAD_CUDA_THREADS), TV_GRAD_CUDA_THREADS, 0, (cudaStream_t)stream>>>(
        PackedVar32<int32_t, 3>(&l), PackedVar64<float, 2>(&dv), rand_cells, 0, dim, scale, Q, ignore_edge != 0, false, nullptr, grad);
    return (int)cudaGetLastError();
}
