// clippy_adagrad.cu -- K7: ClippyAdagrad (experimental/optimizers/clippy_adagrad.py:81-249): Adagrad whose step is
// scaled, per variable, by the largest factor in [0, 1] that keeps every touched element's change under
// |v| * var_rel + p * acc_rel + abs_thr.  The factor is a minimum over the whole variable, so every update waits for a
// reduction over all touched elements: pass A computes the factor, pass B applies it.
//   sparse (one embedding table per call): K4's id grouping (ag_group) and run-summing pattern (ag_run_sums).  Pass A
//     sums each run's duplicate rows in order of occurrence, saves the summed row in the workspace (slot = the run's first
//     sorted position) and folds the run's per-element ratios into the factor; pass B updates every run head's row from
//     the saved sum.  Pass A only reads the table and accumulator, pass B does every write.
//   dense (all dense variables of one optimizer): the multi-tensor launches of multi_tensor.cuh (descriptors by value in
//     the kernel parameters, up to CD_MAX variables per launch); one init, one pass A and one pass B launch per batch.
// The factor is an atomicMin on the bit pattern of a non-negative float: a minimum is order-independent, so the result is
// bitwise reproducible.  NaN ratios do not lower it (fminf).  Every arithmetic step is a single IEEE fp32 op (no FMA
// contraction), stated identically by the fp32 restatement the tests use (tests/, clippy_oracle).
// HBM bytes, sparse: pass A  n*d*4 (grads) + 2*u*d*4 (var, acc) + u*d*4 (summed rows written), u = unique rows;
//                    pass B  3*u*d*4 (summed rows, var, acc) + 2*u*d*4 (var, acc written).
//            dense:  pass A  3*N*4 ; pass B  3*N*4 + 2*N*4, N = elements of all variables.
#include "adagrad.cuh"
#include "multi_tensor.cuh"

namespace tfrs {

enum { CL_CLIP_ACCUMULATOR_UPDATE = 1, CL_STANDARD_ACCUMULATOR_UPDATE = 2 };

struct ClippyArgs { float lr, eps, var_rel, acc_rel, abs_thr; int flags; };

// The element rule.  a1 = standard ? a + g*g : a ;  p = 1 / sqrt(a1 + eps) ;  delta = (lr*g) * p ;
// m = (abs_thr + |v|*var_rel) + p*acc_rel ;  ratio = delta == 0 ? 1 : m / |delta|
__device__ __forceinline__ float cl_delta(float g, float a, const ClippyArgs& k, float& a1, float& p) {
  a1 = (k.flags & CL_STANDARD_ACCUMULATOR_UPDATE) ? __fadd_rn(a, __fmul_rn(g, g)) : a;
  p = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(a1, k.eps)));
  return __fmul_rn(__fmul_rn(k.lr, g), p);
}
__device__ __forceinline__ float cl_ratio(float g, float v, float a, const ClippyArgs& k) {
  float a1, p;
  const float delta = cl_delta(g, a, k, a1, p);
  const float m = __fadd_rn(__fadd_rn(k.abs_thr, __fmul_rn(fabsf(v), k.var_rel)), __fmul_rn(p, k.acc_rel));
  return delta == 0.f ? 1.f : __fdiv_rn(m, fabsf(delta));
}
// v' = v - delta*scale ;  a' = standard ? a1 : a + u*u,  u = clip_accumulator_update ? g*scale : g
__device__ __forceinline__ void cl_apply(float g, float& v, float& a, const ClippyArgs& k, float scale) {
  float a1, p;
  const float delta = cl_delta(g, a, k, a1, p);
  v = __fsub_rn(v, __fmul_rn(delta, scale));
  if (k.flags & CL_STANDARD_ACCUMULATOR_UPDATE) {
    a = a1;
  } else {
    const float u = (k.flags & CL_CLIP_ACCUMULATOR_UPDATE) ? __fmul_rn(g, scale) : g;
    a = __fadd_rn(a, __fmul_rn(u, u));
  }
}
// min over the warp, then one atomicMin per warp (skipped when nothing is below 1, the factor's starting value)
__device__ __forceinline__ void cl_fold_min(float m, float* factor) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m < 1.f) atomicMin(reinterpret_cast<unsigned int*>(factor), __float_as_uint(m));
}

__global__ void cl_fill_one(float* __restrict__ f, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f[i] = 1.f;
}

// ---- sparse ----------------------------------------------------------------------------------------------------------
// Pass A as the epilogue of K4's run-summing kernels: save the summed row, fold its ratios into the factor.
struct ClippyFactorOp {
  const float* table; const float* accum; float* sums; float* factor; ClippyArgs k;
  struct State { float m = 1.f; };
  __device__ __forceinline__ void column(State& s, long long row, long long head, int d, int c, float g) const {
    sums[head * d + c] = g;
    const long long e = row + c;
    s.m = fminf(s.m, cl_ratio(g, table[e], accum[e], k));
  }
  __device__ __forceinline__ void finish(State& s) const { cl_fold_min(s.m, factor); }
};

// Pass B: one warp per run head, the summed row from pass A
__global__ void __launch_bounds__(256)
cl_sparse_apply(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ sums, int d,
                float* __restrict__ table, float* __restrict__ accum, const float* __restrict__ factor, const ClippyArgs k) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  unsigned long long id;
  if (i >= n || !ag_run_head(keys, i, id)) return;
  const float scale = *factor;
  float* trow = table + (long long)id * d;
  float* arow = accum + (long long)id * d;
  for (int c = lane; c < d; c += 32) {
    float v = trow[c], a = arow[c];
    cl_apply(sums[i * d + c], v, a, k, scale);
    trow[c] = v; arow[c] = a;
  }
}

// ---- dense -----------------------------------------------------------------------------------------------------------
// 32 B per descriptor + 4 B of block offset: 896 variables and the scalars stay under the 32764 bytes of kernel
// parameters that CUDA 12.1+ allows on sm_90.
constexpr int CD_MAX = 896;
struct CdVar { float* var; const float* grad; float* acc; long long numel; };
using CdBatch = MtBatch<CdVar, CD_MAX>;
static_assert(sizeof(CdBatch) + sizeof(ClippyArgs) + 2 * sizeof(void*) <= 32764, "kernel parameters over the sm_90 limit");

__global__ void __launch_bounds__(MT_THREADS)
cl_dense_factor(const __grid_constant__ CdBatch b, const ClippyArgs k, float* __restrict__ factors) {
  const int v = mt_find(b);
  const CdVar& x = b.v[v];
  const long long e0 = mt_first(b, v);
  float m = 1.f;
#pragma unroll
  for (int u = 0; u < MT_PER_THREAD; ++u) {
    const long long e = e0 + u * MT_THREADS;
    if (e < x.numel) m = fminf(m, cl_ratio(x.grad[e], x.var[e], x.acc[e], k));
  }
  cl_fold_min(m, factors + v);
}

__global__ void __launch_bounds__(MT_THREADS)
cl_dense_apply(const __grid_constant__ CdBatch b, const ClippyArgs k, const float* __restrict__ factors) {
  const int v = mt_find(b);
  const CdVar& x = b.v[v];
  const float scale = factors[v];
  const long long e0 = mt_first(b, v);
#pragma unroll
  for (int u = 0; u < MT_PER_THREAD; ++u) {
    const long long e = e0 + u * MT_THREADS;
    if (e < x.numel) {
      float val = x.var[e], a = x.acc[e];
      cl_apply(x.grad[e], val, a, k, scale);
      x.var[e] = val; x.acc[e] = a;
    }
  }
}

// -0.0 thresholds become +0.0, so that no ratio is -0.0 (whose bit pattern would not order below 1.0f)
static int cl_args(float lr, float eps, float var_rel, float acc_rel, float abs_thr, int flags, ClippyArgs* k) {
  TFRS_CHECK_ARG(var_rel >= 0.f && acc_rel >= 0.f && abs_thr >= 0.f,
                 "clippy_adagrad: variable / accumulator relative and absolute thresholds must be non-negative");
  TFRS_CHECK_ARG(flags >= 0 && flags <= 3 && flags != 3,
                 "clippy_adagrad: flags must be a subset of {1: clip_accumulator_update, 2: use_standard_accumulator_update}, "
                 "not both");
  *k = ClippyArgs{lr, eps, var_rel + 0.f, acc_rel + 0.f, abs_thr + 0.f, flags};
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_sparse_clippy_adagrad_workspace_bytes(int64_t n, int d) {
  const size_t nn = n > 0 ? (size_t)n : 0, dd = d > 0 ? (size_t)d : 0;
  return align_up(ag_group_workspace_bytes(n), 256) + align_up(nn * dd * 4, 256) + 256;
}

extern "C" int tfrs_sparse_clippy_adagrad_f32(float* table, float* accum, int64_t rows, int d, const void* ids, int ids_dtype,
                                              int64_t n, const float* grad_rows, float lr, float eps, float var_rel,
                                              float acc_rel, float abs_thr, int flags, float* clipping_factor_out, void* ws,
                                              size_t ws_bytes, void* stream) {
  int rc;
  if ((rc = ag_check_args("sparse_clippy_adagrad", table && accum, rows, d, ids_dtype, n, ids, grad_rows)) != TFRS_OK) return rc;
  TFRS_CHECK_ARG(d <= 1024, "sparse_clippy_adagrad: d=%d > 1024", d);
  ClippyArgs k;
  rc = cl_args(lr, eps, var_rel, acc_rel, abs_thr, flags, &k);
  if (rc != TFRS_OK) return rc;
  if (!ws || ws_bytes < tfrs_sparse_clippy_adagrad_workspace_bytes(n, d)) {
    set_error("sparse_clippy_adagrad: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = (float*)((char*)ws + align_up(ag_group_workspace_bytes(n), 256));
  float* factor = clipping_factor_out ? clipping_factor_out : (float*)((char*)sums + align_up((size_t)n * d * 4, 256));
  cl_fill_one<<<1, 32, 0, st>>>(factor, 1);   // no touched element: factor 1
  TFRS_LAUNCH_CHECK();
  if (n == 0) return TFRS_OK;
  AgGroups gr;
  if ((rc = ag_group(ids, ids_dtype, n, rows, ws, st, &gr)) != TFRS_OK) return rc;
  if ((rc = ag_run_sums(gr, n, grad_rows, d, ClippyFactorOp{table, accum, sums, factor, k}, st)) != TFRS_OK) return rc;
  cl_sparse_apply<<<(unsigned)ceil_div(n * 32, 256), 256, 0, st>>>(gr.keys, n, sums, d, table, accum, factor, k);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_clippy_adagrad_dense_workspace_bytes(int nvars) {
  return align_up((size_t)(nvars > 0 ? nvars : 0) * 4, 256) + 256;
}

extern "C" int tfrs_clippy_adagrad_dense_f32(float* const* vars, const float* const* grads, float* const* accums,
                                             const int64_t* numels, int nvars, float lr, float eps, float var_rel,
                                             float acc_rel, float abs_thr, int flags, float* clipping_factors_out, void* ws,
                                             size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(nvars >= 0, "clippy_adagrad_dense: nvars=%d < 0", nvars);
  if (nvars == 0) return TFRS_OK;
  TFRS_CHECK_ARG(vars && grads && accums && numels, "clippy_adagrad_dense: NULL descriptor array");
  for (int i = 0; i < nvars; ++i) {
    TFRS_CHECK_ARG(numels[i] >= 0 && numels[i] < (1ll << 40), "clippy_adagrad_dense: numel[%d]=%lld out of range", i,
                   (long long)numels[i]);
    TFRS_CHECK_ARG(numels[i] == 0 || (vars[i] && grads[i] && accums[i]), "clippy_adagrad_dense: NULL pointer for variable %d", i);
  }
  ClippyArgs k;
  const int rc = cl_args(lr, eps, var_rel, acc_rel, abs_thr, flags, &k);
  if (rc != TFRS_OK) return rc;
  if (!clipping_factors_out && (!ws || ws_bytes < tfrs_clippy_adagrad_dense_workspace_bytes(nvars))) {
    set_error("clippy_adagrad_dense: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* factors = clipping_factors_out ? clipping_factors_out : (float*)ws;
  cl_fill_one<<<(unsigned)ceil_div(nvars, 256), 256, 0, st>>>(factors, nvars);
  TFRS_LAUNCH_CHECK();
  return mt_for_each_batch<CdVar, CD_MAX>(
      nvars, numels, "clippy_adagrad_dense",
      [&](int v) { return CdVar{vars[v], grads[v], accums[v], numels[v]}; },
      [&](const CdBatch& b, unsigned blocks, int v0) {
        cl_dense_factor<<<blocks, MT_THREADS, 0, st>>>(b, k, factors + v0);
        TFRS_LAUNCH_CHECK();
        cl_dense_apply<<<blocks, MT_THREADS, 0, st>>>(b, k, factors + v0);
        TFRS_LAUNCH_CHECK();
        return TFRS_OK;
      });
}
