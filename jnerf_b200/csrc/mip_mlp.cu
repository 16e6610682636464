// Mip-NeRF's MipNerfMLP (models/networks/mip_network.py:124-216 of the reference's contrib/mipnerf) on the vanilla NeRF forward kernel of
// nerf_mlp.cuh: the same 8x256 trunk with its skip, density / bottleneck / view / colour layers and the same flat fp16 parameter layout,
// with the integrated positional encoding of the cone-cast intervals as its encode stage.  The backward is nerf_mlp.cu's (ngp_nerf_bwd):
// it reads only the saved layer inputs, whose layout does not depend on the encoder.  DESIGN.md section 11.
#include "mip_common.cuh"
#include "nerf_mlp.cuh"

namespace nerf {
// in = rays (R, 12), stride = S: tile row `row` is interval row % S of ray row / S, between fenceposts t[ray][i] and t[ray][i + 1] (t is
// (R, S + 1)).  pos(): the 48 IPE columns in the reference's order [sin | cos], deg-major, xyz inner, zero to 64; rows at or past n
// encode mean 0, variance 0.  dir(): FrequencyEncoder(4) of the ray's viewdir in the kernel's own order; plugin/mip.py permutes the
// view layer's columns to the reference's pos_enc order.
struct MipEnc {
    const float* t;
    uint32_t cylinder, integrate;
    int min_deg;
    __device__ __forceinline__ void pos(uint8_t* slab, const float* rays, uint32_t S, uint32_t row0, uint32_t n, uint32_t tid) const {
        for (uint32_t k = tid; k < ROWS * 3; k += THREADS) {
            const uint32_t r = k / 3, dim = k % 3, row = row0 + r;
            auto put = [&](uint32_t f, float v) { *reinterpret_cast<__half*>(slab + (f / 8) * GB + r * 16 + (f % 8) * 2) = __float2half_rn(v); };
            float mean = 0.f, var = 0.f;
            if (row < n) {
                const uint32_t ray = row / S, i = row % S;
                const float* tt = t + (size_t)ray * (S + 1) + i;
                mip::gaussian(rays + (size_t)ray * mip::RAY_FLOATS, tt[0], tt[1], dim, cylinder, integrate, mean, var);
            }
            mip::ipe(mean, var, dim, min_deg, put);
            if (dim == 0)
                for (uint32_t f = mip::IPE_W; f < 64; ++f) put(f, 0.f);
        }
    }
    __device__ __forceinline__ void dir(uint8_t* slab, const float* rays, uint32_t S, uint32_t row0, uint32_t n, uint32_t tid) const {
        encode_rows<mip::VIEW_DEGS>(slab, [&](uint32_t row, uint32_t dim) { return rays[(size_t)(row / S) * mip::RAY_FLOATS + 6 + dim]; }, row0, n, tid);
    }
};
}  // namespace nerf

using namespace nerf;

extern "C" int ngp_mip_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate,
                           int min_deg, const void* params, void* out, void* saved) {
    NGP_REQUIRE(n_samples > 0 && (uint64_t)n_rays * n_samples < (1ull << 32), "ngp_mip_fwd: n_samples must be > 0 and n_rays * n_samples < 2^32");
    NGP_REQUIRE(ray_shape == 0 || ray_shape == 1, "ngp_mip_fwd: ray_shape must be 0 (cone) or 1 (cylinder)");
    const uint32_t n = n_rays * n_samples;
    if (n == 0) return 0;
    NGP_REQUIRE(rays && t && params && out, "ngp_mip_fwd: NULL input");
    NGP_REQUIRE(((uintptr_t)params & 15) == 0 && ((uintptr_t)saved & 15) == 0, "ngp_mip_fwd: params / saved must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const MipEnc enc{t, (uint32_t)ray_shape, (uint32_t)(integrate != 0), min_deg};
    return saved ? launch_fwd<false, true>(s, n, nullptr, rays, n_samples, params, out, saved, enc)
                 : launch_fwd<false, false>(s, n, nullptr, rays, n_samples, params, out, nullptr, enc);
}
