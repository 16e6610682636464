// Link-level compatibility with the one native boundary the reference already has (SURVEY.md 8b): the two C++ functions of the
// prebuilt tiny-cuda-nn object `OPS/op_header/fully_fused_mlp_function.o`, declared in OPS/op_header/fully_fused_mlp_header.h:26-60
// and called from the jt.code bodies of OPS/fully_fused_mlp.py:58-75 (forward) and :101-115 (backward).  That object carries
// sm_75/80/86 SASS only and cannot load on an H100; exporting the same two MANGLED symbols from libngp_b200.so lets
// fully_fused_mlp.py link unchanged (`-Xlinker <path to libngp_b200.so>` in place of the .o, INTEGRATION.md section 3).
//
// Contract taken from the call sites (the object has no source in the reference tree):
//   forward : input (B,32) fp16 row-major, B a multiple of 128 (:78-82 pads); weights flat, each layer (out,in) row-major,
//             last layer padded to 16 outputs (:26-40); output_intermediate ((n_hidden_layers+1)*B, 64): block k = post-ReLU
//             activations of hidden layer k (:133-142); output (B,16), no output activation.
//   backward: dL_doutput (16,B) feature-major (grads.transpose(), :117); temps ((n_hidden_matmuls+1)*B, 64) in REVERSE layer
//             order (block 0 = gradient at the last hidden layer, :127-142); weights = weights_first_layer + 64*32 (:106);
//             dL_dinput is written only when need_last (the reference sets it only for 64-wide inputs, :100, never for NGP).
//   errors  : C++ exceptions (std::runtime_error), like the object ("not supported WIDTH=", "Batch size must be a multiple of").
// The weight gradients are NOT part of this symbol pair (the reference computes them with five cuBLAS GEMMs, :123-143);
// ngp_mlp_bwd (include/ngp_b200.h) is the entry point that also returns them from the same kernel.
#include "ngp_common.cuh"
#include "../../include/ngp_b200.h"
#include <cuda_fp16.h>
#include <stdexcept>
#include <string>

// Same global-scope type name and enumerator order as fully_fused_mlp_header.h:19-27: the mangled symbol names contain
// "10Activation", and the call sites pass Activation::ReLU (0) / Activation::None (6).
typedef enum Activation { ReLU, Exponential, Sine, Sigmoid, Squareplus, Softplus, None } Activation;

namespace {
void require(bool ok, const std::string& what) {
    if (!ok) throw std::runtime_error(what);
}
void check_rc(int rc, const char* who) {
    if (rc != 0) throw std::runtime_error(std::string(who) + ": " + ngp_last_error());
}
}  // namespace

void mlp_fused_forward_func(int WIDTH, Activation ACTIVATION, bool INFERENCE, cudaStream_t stream, Activation output_activation,
                            __half* weights, __half* input, __half* output_intermediate, __half* output, const uint32_t n_hidden_layers,
                            int input_shape0, int input_shape1, int weights_shape0, int weights_shape1, int output_shape0, int output_shape1) {
    require(WIDTH == 64, "not supported WIDTH=" + std::to_string(WIDTH) + " (libngp_b200: 64 only)");
    require(ACTIVATION == ReLU && output_activation == None, "libngp_b200 mlp_fused_forward_func: ReLU hidden / None output activation only");
    require(input_shape1 == 32 && weights_shape0 == 32 && weights_shape1 == 64 && output_shape1 == 16,
            "libngp_b200 mlp_fused_forward_func: built for 32 -> 64 (x k) -> 16");
    require(input_shape0 >= 0 && input_shape0 == output_shape0 && input_shape0 % 128 == 0,
            "Batch size must be a multiple of 128 (got " + std::to_string(input_shape0) + ")");
    require(n_hidden_layers <= 3, "libngp_b200 mlp_fused_forward_func: at most 3 hidden matmuls");
    check_rc(ngp_mlp_fwd((void*)stream, weights, input, INFERENCE ? nullptr : output_intermediate, output, n_hidden_layers, (uint32_t)input_shape0),
             "mlp_fused_forward_func");
}

void mlp_fused_backward_func(int WIDTH, Activation ACTIVATION, cudaStream_t stream, __half* weights_first_layer, __half* weights,
                             __half* dL_doutput, __half* temps, __half* forward, __half* dL_dinput, const uint32_t n_hidden_matmuls,
                             int grad_shape0, int grad_shape1, int need_last) {
    require(WIDTH == 64, "not supported WIDTH=" + std::to_string(WIDTH) + " (libngp_b200: 64 only)");
    require(ACTIVATION == ReLU, "libngp_b200 mlp_fused_backward_func: ReLU only");
    require(grad_shape1 == 16, "libngp_b200 mlp_fused_backward_func: dL_doutput must be (16, batch) feature-major");
    require(grad_shape0 >= 0 && grad_shape0 % 128 == 0, "Batch size must be a multiple of 128 (got " + std::to_string(grad_shape0) + ")");
    require(weights == weights_first_layer + 64 * 32, "libngp_b200 mlp_fused_backward_func: weights must follow a 32x64 first layer in one flat buffer");
    require(!need_last, "libngp_b200 mlp_fused_backward_func: need_last is for 64-wide inputs (not an NGP configuration)");
    require(n_hidden_matmuls <= 3, "libngp_b200 mlp_fused_backward_func: at most 3 hidden matmuls");
    (void)dL_dinput;
    check_rc(ngp_mlp_bwd_dgrad((void*)stream, weights_first_layer, forward, dL_doutput, nullptr, temps, n_hidden_matmuls, (uint32_t)grad_shape0),
             "mlp_fused_backward_func");
}
