// stub for Jittor's var.h (Jittor is not installed): the Plenoxels headers (jt_helper.h, data_spec.h) only read a Var's data
// pointer, shape and element count.
#pragma once
#include <cstdint>
namespace jittor {
struct Var {
    void* mem;
    int64_t shape[4];
    int64_t num;
    template <class T> T* ptr() { return static_cast<T*>(mem); }
};
}  // namespace jittor
