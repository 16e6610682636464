// The u32 exclusive scan of mesh.cu, also used by mesh_smooth.cu to number the band variables in lattice order.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace ngp_mesh {
constexpr uint32_t SCAN_BLOCK = 2048;   // elements per block: bsum needs ceil(len / SCAN_BLOCK) entries
// a[0..len) -> its exclusive prefix sums, in place; the sum -> *total (device).  Three launches, no host sync.
int scan_u32(cudaStream_t s, uint32_t* a, uint32_t len, uint32_t* bsum, uint32_t* total);
}  // namespace ngp_mesh
