// Error state, version and small host-side helpers of the C ABI (include/ngp_b200.h).
#include "ngp_common.cuh"
#include <cuda.h>
#include <vector>
#include <utility>
#include <mutex>

namespace {
std::mutex g_err_mu;
thread_local std::string g_err;
}  // namespace

void ngp_set_error(const std::string& msg) { g_err = msg; }

int ngp_num_sms() {
    static int sms[64] = {0};                                     // per device: a process may drive several GPUs
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (sms[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
        sms[dev] = n;
    }
    return sms[dev];
}

// Tensor map for the encoded-feature matrix (rows, 32) fp16: box = 8 columns (one slab feature group) x 128 rows (one tile).
// cuTensorMapEncodeTiled is a driver entry point; the library links the runtime only, so it is looked up through the runtime.
bool ngp_make_rows32_tensormap(NgpTensorMap* out, const void* base, unsigned long long n_rows) {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    static bool looked = false;
    if (!looked) {
        looked = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeFn)p;
    }
    if (!fn || n_rows == 0 || (reinterpret_cast<uintptr_t>(base) & 15)) return false;
    static_assert(sizeof(NgpTensorMap) == sizeof(CUtensorMap), "tensor map size");
    const cuuint64_t dims[2] = {32, n_rows};
    const cuuint64_t strides[1] = {64};                          // bytes between rows
    const cuuint32_t box[2] = {8, 128}, estr[2] = {1, 1};
    return fn(reinterpret_cast<CUtensorMap*>(out), CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) instead of on every launch
bool ngp_first_use(const void* kernel) {
    static std::vector<std::pair<const void*, int>> seen;
    int dev = 0;
    cudaGetDevice(&dev);
    for (const auto& e : seen)
        if (e.first == kernel && e.second == dev) return false;
    seen.emplace_back(kernel, dev);
    return true;
}

extern "C" {

const char* ngp_last_error(void) { return g_err.c_str(); }
int ngp_version(void) { return 100; }
int ngp_sm_count(void) { return ngp_num_sms(); }

// ops/op_include/pcg32/pcg32.h:53-60 (seed) and :145-166 (advance); pure integer, host side
void ngp_pcg32_seed(uint64_t initstate, uint64_t initseq, uint64_t* state_inc) {
    Pcg32 r;
    r.state = 0;
    r.inc = (initseq << 1u) | 1u;
    r.next_uint();
    r.state += initstate;
    r.next_uint();
    state_inc[0] = r.state;
    state_inc[1] = r.inc;
}
void ngp_pcg32_advance(uint64_t* state_inc, int64_t delta) {
    Pcg32 r{state_inc[0], state_inc[1]};
    r.advance(delta);
    state_inc[0] = r.state;
}

}  // extern "C"
