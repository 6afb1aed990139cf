// gru.cuh -- gate arithmetic of the GRU recurrence (K19), shared by its forward and backward kernels (gru.cu).  The
// derivatives are taken from the saved gate OUTPUTS, as TF's SigmoidGrad / TanhGrad do.
#pragma once
#include "dense.cuh"

namespace tfrs {

// 1 / (1 + expf(-x)): the Dense layer's sigmoid
__device__ __forceinline__ float gru_sigmoid(float x) { return dense_act(TFRS_ACT_SIGMOID, x); }
__device__ __forceinline__ float gru_tanh(float x) { return tanhf(x); }
// sigmoid'(x) = s (1 - s) and tanh'(x) = 1 - y^2 from s = sigmoid(x), y = tanh(x)
__device__ __forceinline__ float gru_sigmoid_grad(float s) { return s * (1.f - s); }
__device__ __forceinline__ float gru_tanh_grad(float y) { return 1.f - y * y; }

}  // namespace tfrs
