// oracle/_ref build: the reference's Plenoxels resample kernels (contrib/plenoxel misc_kernel.h: dilate, grid weight render) compiled
// UNMODIFIED for sm_90a, with dilate.py's launch shape.  TEST / BENCH INFRASTRUCTURE: never linked into libngp_b200.so.
#include "misc_kernel.h"

// out (X, Y, Z) bool = the dilation of grid (X, Y, Z) bool
extern "C" int ref_svox_dilate(int X, int Y, int Z, const bool* grid, bool* out, void* stream) {
    jittor::Var g{const_cast<bool*>(grid), {X, Y, Z, 1}, (int64_t)X * Y * Z}, o{out, {X, Y, Z, 1}, (int64_t)X * Y * Z};
    const int Q = X * Y * Z;
    dilate_kernel<<<CUDA_N_BLOCKS_NEEDED(Q, MISC_CUDA_THREADS), MISC_CUDA_THREADS, 0, (cudaStream_t)stream>>>(PackedVar32<bool, 3>(&g),
                                                                                                              PackedVar32<bool, 3>(&o));
    return (int)cudaGetLastError();
}
