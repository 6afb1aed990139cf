// dense.cuh -- activations of the Dense layer (K6), shared by the exact kernels (dense.cu) and the DENSE epilogues of the
// split-fp16 tensor-core GEMM (split_gemm.cu); and the steps of K6's backward that the 1-D convolution (K27) shares.
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

// K6's route rule: the split-fp16 tensor-core GEMM for a [B, K] . [K, N] product when true, the exact CUDA-core kernels else
bool dense_tc(long long B, int K, int N);
// dz = dy * act'(y) + dl over `total` elements (dy or dl nullable), one launch
int dense_dz(const float* y, const float* dy, const float* dl, long long total, int act, float* dz, cudaStream_t st);
// out[n] = sum over the B rows of dz [B, N], in float64 and a fixed order: row splits summed into colpart
// (dense_colsum_bytes(N) bytes), then folded in split order; two launches
size_t dense_colsum_bytes(int N);
int dense_colsum(const float* dz, long long B, int N, double* colpart, float* out, cudaStream_t st);

}  // namespace tfrs
