// sgd.cu -- plain SGD with tf-keras's legacy rules (optimizer_v2/gradient_descent.py, momentum 0):
//   dense:   var' = var - lr*g                                    (_resource_apply_dense: ResourceApplyGradientDescent)
//   sparse:  var[id] -= lr*g_i once per occurrence i of id        (_resource_apply_sparse: resource_scatter_add of
//            -lr*g without deduplication; the order duplicates land in is unpinned, here the order of occurrence)
// Every step is one IEEE fp32 operation: var = __fsub_rn(var, __fmul_rn(lr, g)).
// Sparse (one embedding table per call): K4's id grouping (ag_group) orders the occurrences by (id, position); one warp
//   per run of equal ids then applies the run's rows in order, 8 gradient rows in flight per step.  Out-of-range ids are
//   skipped.  Deterministic, no atomics.
// Dense (all dense variables of one optimizer): the multi-tensor launches of multi_tensor.cuh.
// HBM bytes, sparse: 2*u*d*4 (touched rows read and written) + n*d*4 (grads) + the grouping; dense: 3*N*4.
#include "adagrad.cuh"
#include "multi_tensor.cuh"

namespace tfrs {

__global__ void __launch_bounds__(256)
sgd_sparse_runs(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ grad, int d,
                float* __restrict__ table, float lr) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per sorted slot
  const int lane = threadIdx.x & 31;
  unsigned long long id;
  if (i >= n || !ag_run_head(keys, i, id)) return;
  long long end = i + 1;
  while (end < n && (keys[end] >> 24) == id) ++end;
  float* __restrict__ row = table + (long long)id * d;
  for (int c = lane; c < d; c += 32) {
    float x = row[c];
    for (long long m0 = i; m0 < end; m0 += 8) {
      float g[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        g[u] = m0 + u < end ? __ldg(grad + (long long)(keys[m0 + u] & 0xFFFFFFull) * d + c) : 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (m0 + u < end) x = __fsub_rn(x, __fmul_rn(lr, g[u]));
    }
    row[c] = x;
  }
}

// 32 B per descriptor + 4 B of block offset: 896 variables stay under the 32764 bytes of sm_90 kernel parameters.
constexpr int SGD_MAX = 896;
struct SgdVar { float* var; const float* grad; long long numel; long long pad; };
using SgdBatch = MtBatch<SgdVar, SGD_MAX>;
static_assert(sizeof(SgdBatch) + sizeof(float) <= 32764, "kernel parameters over the sm_90 limit");

__global__ void __launch_bounds__(MT_THREADS)
sgd_dense_apply(const __grid_constant__ SgdBatch b, const float lr) {
  const int vi = mt_find(b);
  const SgdVar& x = b.v[vi];
  const long long e0 = mt_first(b, vi);
#pragma unroll
  for (int u = 0; u < MT_PER_THREAD; ++u) {
    const long long e = e0 + u * MT_THREADS;
    if (e < x.numel) x.var[e] = __fsub_rn(x.var[e], __fmul_rn(lr, x.grad[e]));
  }
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_sparse_sgd_workspace_bytes(int64_t n) { return ag_group_workspace_bytes(n > 0 ? n : 1); }

extern "C" int tfrs_sparse_sgd_f32(float* table, int64_t rows, int d, const void* ids, int ids_dtype, int64_t n,
                                   const float* grad_rows, float lr, void* ws, size_t ws_bytes, void* stream) {
  int rc;
  if ((rc = ag_check_args("sparse_sgd", table, rows, d, ids_dtype, n, ids, grad_rows)) != TFRS_OK) return rc;
  if (n == 0) return TFRS_OK;
  if (!ws || ws_bytes < tfrs_sparse_sgd_workspace_bytes(n)) {
    set_error("sparse_sgd: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  AgGroups gr;
  if ((rc = ag_group(ids, ids_dtype, n, rows, ws, st, &gr)) != TFRS_OK) return rc;
  sgd_sparse_runs<<<(unsigned)ceil_div(n * 32, 256), 256, 0, st>>>(gr.keys, n, grad_rows, d, table, lr);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_sgd_dense_f32(float* const* vars, const float* const* grads, const int64_t* numels, int nvars, float lr,
                                  void* stream) {
  TFRS_CHECK_ARG(nvars >= 0, "sgd_dense: nvars=%d < 0", nvars);
  if (nvars == 0) return TFRS_OK;
  TFRS_CHECK_ARG(vars && grads && numels, "sgd_dense: NULL descriptor array");
  for (int i = 0; i < nvars; ++i) {
    TFRS_CHECK_ARG(numels[i] >= 0 && numels[i] < (1ll << 40), "sgd_dense: numel[%d]=%lld out of range", i,
                   (long long)numels[i]);
    TFRS_CHECK_ARG(numels[i] == 0 || (vars[i] && grads[i]), "sgd_dense: NULL pointer for variable %d", i);
  }
  cudaStream_t st = (cudaStream_t)stream;
  return mt_for_each_batch<SgdVar, SGD_MAX>(
      nvars, numels, "sgd_dense",
      [&](int i) { return SgdVar{vars[i], grads[i], numels[i], 0}; },
      [&](const SgdBatch& b, unsigned blocks, int) {
        sgd_dense_apply<<<blocks, MT_THREADS, 0, st>>>(b, lr);
        TFRS_LAUNCH_CHECK();
        return TFRS_OK;
      });
}
