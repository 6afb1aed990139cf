// adam.cu -- K10: Adam, with tf-keras's legacy rules (optimizer_v2/adam.py: _resource_apply_dense, and
// _resource_apply_sparse for embedding tables).  The host computes alpha = lr * sqrt(1 - b2^t) / (1 - b1^t) once per step;
// omb1 = 1 - b1 and omb2 = 1 - b2 are computed here in fp32.  Every step below is one IEEE fp32 operation (no FMA
// contraction), stated identically by the NumPy float32 restatement the tests use (tests/, adam_oracle).
//   dense:            m' = m + (g - m)*omb1 ;  v' = v + (g*g - v)*omb2 ;  var' = var - (m'*alpha) / (sqrt(v') + eps)
//   sparse, touched:  m' = m*b1 + g*omb1    ;  v' = v*b2 + (g*g)*omb2  ;  var' = var - (alpha*m') / (sqrt(v') + eps)
//   sparse, other rows (not lazy):  m' = m*b1 ;  v' = v*b2 ;  var' as above.  lazy: other rows are not touched at all.
// Sparse (one embedding table per call): K4's id grouping (ag_group) and run-summing kernels (ag_run_sums) with an
//   AdamRowOp epilogue, which sums each id's gradient rows in order of occurrence, updates the row in place and, unless
//   lazy, sets the row's bit in a rows-bit bitmap.  Then (not lazy) one grid-stride pass applies the untouched-row rule to
//   every row whose bit is clear.  The two write sets are disjoint and the launches are ordered on the stream, so the
//   result is deterministic; the decay is never applied first and scattered over, which would cost another pass.
// Dense (all dense variables of one optimizer): the multi-tensor launches of multi_tensor.cuh, one launch per batch.
// HBM bytes, sparse not lazy: 6*rows*d*4 (var, m, v read and written) + n*d*4 (grads) + rows/8 (bitmap);
//            sparse lazy:     6*u*d*4 + n*d*4, u = unique rows;
//            dense:           7*N*4 (var, m, v read and written, grad read), N = elements of all variables.
#include "adagrad.cuh"
#include "multi_tensor.cuh"

namespace tfrs {

struct AdamArgs { float alpha, b1, b2, omb1, omb2, eps; };

// var' = var - (alpha*m') / (sqrt(v') + eps)
__device__ __forceinline__ float ad_var(float var, float m1, float v1, const AdamArgs& k) {
  return __fsub_rn(var, __fdiv_rn(__fmul_rn(k.alpha, m1), __fadd_rn(__fsqrt_rn(v1), k.eps)));
}

// ---- sparse ----------------------------------------------------------------------------------------------------------
// The touched-row rule as the epilogue of K4's run-summing kernels.  `touched` is NULL in lazy mode.
struct AdamRowOp {
  float* table; float* m; float* v; unsigned int* touched; AdamArgs k;
  struct State {};
  __device__ __forceinline__ void column(State&, long long row, long long, int d, int c, float g) const {
    const long long e = row + c;
    const float m1 = __fadd_rn(__fmul_rn(m[e], k.b1), __fmul_rn(g, k.omb1));
    const float v1 = __fadd_rn(__fmul_rn(v[e], k.b2), __fmul_rn(__fmul_rn(g, g), k.omb2));
    m[e] = m1; v[e] = v1;
    table[e] = ad_var(table[e], m1, v1, k);
    if (touched && c == 0) {
      const long long id = row / d;
      atomicOr(touched + (id >> 5), 1u << (id & 31));
    }
  }
  __device__ __forceinline__ void finish(State&) const {}
};

__device__ __forceinline__ void ad_decay(float& var, float& m, float& v, const AdamArgs& k) {
  m = __fmul_rn(m, k.b1);
  v = __fmul_rn(v, k.b2);
  var = ad_var(var, m, v, k);
}

// The untouched-row rule on every row whose bit is clear.  A thread walks the (row, column group) pairs of a grid-stride
// loop by increments, so no element pays a 64-bit division.  V = 4: float4 groups (d % 4 == 0 and table, m and v 16-byte
// aligned), V = 1: single columns.
template <int V>
__global__ void __launch_bounds__(256)
ad_decay_untouched(float* __restrict__ table, float* __restrict__ m, float* __restrict__ v, long long rows, int groups,
                   const unsigned int* __restrict__ touched, const AdamArgs k) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // = row * groups + c
  long long row = e / groups;
  int c = (int)(e - row * groups);
  const long long srow = stride / groups;
  const int sc = (int)(stride - srow * groups);
  for (; row < rows; e += stride) {
    if (!((__ldg(touched + (row >> 5)) >> (row & 31)) & 1u)) {
      if constexpr (V == 4) {
        float4 x = reinterpret_cast<float4*>(table)[e], a = reinterpret_cast<float4*>(m)[e], b = reinterpret_cast<float4*>(v)[e];
        ad_decay(x.x, a.x, b.x, k); ad_decay(x.y, a.y, b.y, k); ad_decay(x.z, a.z, b.z, k); ad_decay(x.w, a.w, b.w, k);
        reinterpret_cast<float4*>(table)[e] = x; reinterpret_cast<float4*>(m)[e] = a; reinterpret_cast<float4*>(v)[e] = b;
      } else {
        float x = table[e], a = m[e], b = v[e];
        ad_decay(x, a, b, k);
        table[e] = x; m[e] = a; v[e] = b;
      }
    }
    row += srow; c += sc;
    if (c >= groups) { c -= groups; ++row; }
  }
}

// ---- dense -----------------------------------------------------------------------------------------------------------
// 40 B per descriptor + 4 B of block offset: 736 variables and the scalars stay under the 32764 bytes of kernel
// parameters that CUDA 12.1+ allows on sm_90.
constexpr int AD_MAX = 736;
struct AdVar { float* var; const float* grad; float* m; float* v; long long numel; };
using AdBatch = MtBatch<AdVar, AD_MAX>;
static_assert(sizeof(AdBatch) + sizeof(AdamArgs) <= 32764, "kernel parameters over the sm_90 limit");

__global__ void __launch_bounds__(MT_THREADS)
ad_dense_apply(const __grid_constant__ AdBatch b, const AdamArgs k) {
  const int vi = mt_find(b);
  const AdVar& x = b.v[vi];
  const long long e0 = mt_first(b, vi);
#pragma unroll
  for (int u = 0; u < MT_PER_THREAD; ++u) {
    const long long e = e0 + u * MT_THREADS;
    if (e < x.numel) {
      const float g = x.grad[e], m = x.m[e], v = x.v[e];
      const float m1 = __fadd_rn(m, __fmul_rn(__fsub_rn(g, m), k.omb1));
      const float v1 = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(g, g), v), k.omb2));
      x.m[e] = m1; x.v[e] = v1;
      x.var[e] = ad_var(x.var[e], m1, v1, k);
    }
  }
}

static AdamArgs ad_args(float alpha, float beta1, float beta2, float eps) {
  return AdamArgs{alpha, beta1, beta2, 1.f - beta1, 1.f - beta2, eps};
}

static size_t ad_bitmap_bytes(long long rows) { return (size_t)ceil_div(rows, 32) * 4; }

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_sparse_adam_workspace_bytes(int64_t n, int64_t rows) {
  return align_up(ag_group_workspace_bytes(n), 256) + align_up(ad_bitmap_bytes(rows > 0 ? rows : 0), 256);
}

extern "C" int tfrs_sparse_adam_f32(float* table, float* m, float* v, int64_t rows, int d, const void* ids, int ids_dtype,
                                    int64_t n, const float* grad_rows, float alpha, float beta1, float beta2, float eps,
                                    int lazy, void* ws, size_t ws_bytes, void* stream) {
  int rc;
  if ((rc = ag_check_args("sparse_adam", table && m && v, rows, d, ids_dtype, n, ids, grad_rows)) != TFRS_OK) return rc;
  TFRS_CHECK_ARG(d <= 1024, "sparse_adam: d=%d > 1024", d);
  if (!ws || ws_bytes < tfrs_sparse_adam_workspace_bytes(n, rows)) {
    set_error("sparse_adam: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const AdamArgs k = ad_args(alpha, beta1, beta2, eps);
  unsigned int* touched = lazy ? nullptr : (unsigned int*)((char*)ws + align_up(ag_group_workspace_bytes(n), 256));
  if (touched) TFRS_CUDA(cudaMemsetAsync(touched, 0, ad_bitmap_bytes(rows), st));
  if (n > 0) {
    AgGroups gr;
    if ((rc = ag_group(ids, ids_dtype, n, rows, ws, st, &gr)) != TFRS_OK) return rc;
    if ((rc = ag_run_sums(gr, n, grad_rows, d, AdamRowOp{table, m, v, touched, k}, st)) != TFRS_OK) return rc;
  }
  if (touched) {
    // float4 groups only when table, m and v all start on a 16-byte boundary (a contiguous view need not)
    const bool aligned = ((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    const int V = (d & 3) == 0 && aligned ? 4 : 1;
    const unsigned grid = elementwise_grid(rows * (d / V));
    if (V == 4) ad_decay_untouched<4><<<grid, 256, 0, st>>>(table, m, v, rows, d / 4, touched, k);
    else ad_decay_untouched<1><<<grid, 256, 0, st>>>(table, m, v, rows, d, touched, k);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}

extern "C" int tfrs_adam_dense_f32(float* const* vars, const float* const* grads, float* const* ms, float* const* vs,
                                   const int64_t* numels, int nvars, float alpha, float beta1, float beta2, float eps,
                                   void* stream) {
  TFRS_CHECK_ARG(nvars >= 0, "adam_dense: nvars=%d < 0", nvars);
  if (nvars == 0) return TFRS_OK;
  TFRS_CHECK_ARG(vars && grads && ms && vs && numels, "adam_dense: NULL descriptor array");
  for (int i = 0; i < nvars; ++i) {
    TFRS_CHECK_ARG(numels[i] >= 0 && numels[i] < (1ll << 40), "adam_dense: numel[%d]=%lld out of range", i,
                   (long long)numels[i]);
    TFRS_CHECK_ARG(numels[i] == 0 || (vars[i] && grads[i] && ms[i] && vs[i]), "adam_dense: NULL pointer for variable %d", i);
  }
  cudaStream_t st = (cudaStream_t)stream;
  const AdamArgs k = ad_args(alpha, beta1, beta2, eps);
  return mt_for_each_batch<AdVar, AD_MAX>(
      nvars, numels, "adam_dense",
      [&](int i) { return AdVar{vars[i], grads[i], ms[i], vs[i], numels[i]}; },
      [&](const AdBatch& b, unsigned blocks, int) {
        ad_dense_apply<<<blocks, MT_THREADS, 0, st>>>(b, k);
        TFRS_LAUNCH_CHECK();
        return TFRS_OK;
      });
}
