// The density lattice of vanilla NeRF for mesh extraction (tools/extract_mesh.py:42-70 of the reference, which queries
// runner.model(pos, dir)[:, -1]; OriginNeRFNetworks.density, ori_nerf_network.py:58-67): the density forward of nerf_mlp.cuh with an
// encode stage that makes each row's lattice position itself and an epilogue that stores float(int(max(alpha_raw, 0))) as fp32.
// Its own translation unit, as mip_mlp.cu is: same kernel template, same weight stream, same parameter layout.  DESIGN.md section 4.
#include "nerf_mlp.cuh"

#include <string>

namespace nerf {
// Row r = (i*n + j)*n + k is the model position (i, j, k) / (n-1), each coordinate an IEEE fp32 quotient: the positions a coordinate
// buffer would hold for ngp_nerf_density, so alpha_raw is the same bit for bit.  n <= 1024 keeps r, n*n and every tile index in 32 bits.
struct LatticeEnc {
    static constexpr uint32_t EG = 8;
    uint32_t side;
    __device__ __forceinline__ float coord(uint32_t r, uint32_t dim) const {
        const uint32_t idx = dim == 0 ? r / (side * side) : dim == 1 ? (r / side) % side : r % side;
        return __fdiv_rn((float)idx, (float)(side - 1));
    }
    __device__ __forceinline__ void pos(uint8_t* slab, const float*, uint32_t, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<10>(slab, [&](uint32_t row, uint32_t dim) { return coord(row, dim); }, row0, n, tid);
    }
    __device__ __forceinline__ void dir(uint8_t*, const float*, uint32_t, uint32_t, uint32_t, uint32_t) const {}
    // extract_mesh.py:68: jt.maximum(sigma, 0).int(), kept as float for marching cubes
    __device__ __forceinline__ void store_density(__half* out, uint32_t row, __half alpha) const {
        reinterpret_cast<float*>(out)[row] = truncf(fmaxf(__half2float(alpha), 0.f));
    }
};
}  // namespace nerf

using namespace nerf;

extern "C" int ngp_nerf_density_lattice(void* stream, uint32_t n, const void* params, float* field_out) {
    NGP_REQUIRE(n >= 2 && n <= 1024, "ngp_nerf_density_lattice: resolution n must be in [2, 1024], got " + std::to_string(n));
    NGP_REQUIRE(params && field_out, "ngp_nerf_density_lattice: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0, "ngp_nerf_density_lattice: params must be 16-byte aligned");
    return launch_fwd<true, false>((cudaStream_t)stream, n * n * n, nullptr, nullptr, 0, params, field_out, nullptr, LatticeEnc{n});
}
