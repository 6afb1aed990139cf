// dense.cuh -- activations of the Dense layer (K6), shared by the exact kernels (dense.cu) and the DENSE epilogues of the
// split-fp16 tensor-core GEMM (split_gemm.cu).
#pragma once
#include "common.cuh"

namespace tfrs {

// y = act(z):  TFRS_ACT_LINEAR / RELU / SIGMOID (include/tfrs_b200.h)
__device__ __forceinline__ float dense_act(int act, float z) {
  if (act == TFRS_ACT_RELU) return z > 0.f ? z : 0.f;
  if (act == TFRS_ACT_SIGMOID) return 1.f / (1.f + expf(-z));
  return z;
}

// act'(z) expressed through the saved OUTPUT y (no pre-activation is kept): relu' = [y > 0], sigmoid' = y (1 - y)
// (TF's ReluGrad / SigmoidGrad)
__device__ __forceinline__ float dense_act_grad(int act, float y, float g) {
  if (act == TFRS_ACT_RELU) return y > 0.f ? g : 0.f;
  if (act == TFRS_ACT_SIGMOID) return g * y * (1.f - y);
  return g;
}

}  // namespace tfrs
