// ftrl.cu -- K12: FTRL-Proximal with tf-keras's legacy rules (optimizer_v2/ftrl.py: _resource_apply_dense and, for
// embedding tables, _resource_apply_sparse; TF's ApplyFtrl / ApplyFtrlV2 and their sparse forms).  The host folds beta
// into l2 once per call (l2a = l2 + beta / (2*lr), fp32).  Every step below is one IEEE fp32 operation (no FMA
// contraction), stated identically by the NumPy float32 restatement the tests use (tests/, ftrl_oracle).
//   P(x) = sqrt(x) when lr_power == -0.5 (FT_SQRT), else f32(pow(f64(x), -f64(lr_power))) (FT_POW, rounded once)
//   gs = l2_shrinkage > 0 ? g + (2*l2_shrinkage)*var : g ;  na = acc + g*g
//   lin' = lin + (gs - ((P(na) - P(acc)) / lr)*var) ;  y = P(na)/lr + 2*l2a
//   var' = |lin'| > l1 ? (copysign(l1, lin') - lin') / y : +0 ;  acc' = na
// Sparse (one embedding table per call): K4's id grouping (ag_group) and run-summing kernels (ag_run_sums) with an
//   FtrlRowOp epilogue, which sums each id's gradient rows in order of occurrence and updates the row in place.  Rows no
//   id touches are not read or written.
// Dense (all dense variables of one optimizer): the multi-tensor launches of multi_tensor.cuh, one launch per batch.
// HBM bytes, sparse: 6*u*d*4 (var, acc, lin of the u unique in-range rows read and written) + n*d*4 (grads);
//            dense:  7*N*4 (var, acc, lin read and written, grad read), N = elements of all variables.
#include <cmath>

#include "adagrad.cuh"
#include "multi_tensor.cuh"

namespace tfrs {

enum FtMode { FT_SQRT = 0, FT_POW = 1 };

struct FtrlArgs {
  double neg_power;   // -lr_power (FT_POW)
  float lr, l1, two_l2a, two_shrink;
  int shrink;         // l2_shrinkage > 0
};

template <int MODE>
__device__ __forceinline__ float ft_power(float x, const FtrlArgs& k) {
  if constexpr (MODE == FT_SQRT) return __fsqrt_rn(x);
  else return __double2float_rn(pow((double)x, k.neg_power));
}

template <int MODE>
__device__ __forceinline__ void ft_update(float& var, float& acc, float& lin, float g, const FtrlArgs& k) {
  const float gs = k.shrink ? __fadd_rn(g, __fmul_rn(k.two_shrink, var)) : g;
  const float na = __fadd_rn(acc, __fmul_rn(g, g));
  const float pn = ft_power<MODE>(na, k), pa = ft_power<MODE>(acc, k);
  const float l = __fadd_rn(lin, __fsub_rn(gs, __fmul_rn(__fdiv_rn(__fsub_rn(pn, pa), k.lr), var)));
  const float y = __fadd_rn(__fdiv_rn(pn, k.lr), k.two_l2a);
  var = fabsf(l) > k.l1 ? __fdiv_rn(__fsub_rn(copysignf(k.l1, l), l), y) : 0.f;
  acc = na;
  lin = l;
}

// ---- sparse ----------------------------------------------------------------------------------------------------------
// The element rule as the epilogue of K4's run-summing kernels.
template <int MODE>
struct FtrlRowOp {
  float* table; float* acc; float* lin; FtrlArgs k;
  struct State {};
  __device__ __forceinline__ void column(State&, long long row, long long, int, int c, float g) const {
    const long long e = row + c;
    float x = table[e], a = acc[e], z = lin[e];
    ft_update<MODE>(x, a, z, g, k);
    table[e] = x; acc[e] = a; lin[e] = z;
  }
  __device__ __forceinline__ void finish(State&) const {}
};

// ---- dense -----------------------------------------------------------------------------------------------------------
// 40 B per descriptor + 4 B of block offset: 736 variables and the scalars stay under the 32764 bytes of kernel
// parameters that CUDA 12.1+ allows on sm_90.
constexpr int FT_MAX = 736;
struct FtVar { float* var; const float* grad; float* acc; float* lin; long long numel; };
using FtBatch = MtBatch<FtVar, FT_MAX>;
static_assert(sizeof(FtVar) == 40, "descriptor size");
static_assert(sizeof(FtBatch) + sizeof(FtrlArgs) <= 32764, "kernel parameters over the sm_90 limit");

template <int MODE>
__global__ void __launch_bounds__(MT_THREADS)
ft_dense_apply(const __grid_constant__ FtBatch b, const FtrlArgs k) {
  const int vi = mt_find(b);
  const FtVar& x = b.v[vi];
  const long long e0 = mt_first(b, vi);
#pragma unroll
  for (int u = 0; u < MT_PER_THREAD; ++u) {
    const long long e = e0 + u * MT_THREADS;
    if (e < x.numel) {
      float v = x.var[e], a = x.acc[e], z = x.lin[e];
      ft_update<MODE>(v, a, z, x.grad[e], k);
      x.var[e] = v; x.acc[e] = a; x.lin[e] = z;
    }
  }
}

// The scalar checks shared by both entry points; on success fills *k and returns TFRS_OK.
static int ft_args(const char* what, float lr, float lr_power, float l1, float l2a, float l2_shrinkage, FtrlArgs* k,
                   int* mode) {
  TFRS_CHECK_ARG(std::isfinite(lr) && std::isfinite(lr_power) && std::isfinite(l1) && std::isfinite(l2a) &&
                     std::isfinite(l2_shrinkage), "%s: every scalar must be finite", what);
  TFRS_CHECK_ARG(lr > 0.f, "%s: lr=%g must be > 0", what, (double)lr);
  TFRS_CHECK_ARG(lr_power <= 0.f, "%s: lr_power=%g must be <= 0", what, (double)lr_power);
  TFRS_CHECK_ARG(l1 >= 0.f && l2a >= 0.f && l2_shrinkage >= 0.f, "%s: l1, l2a and l2_shrinkage must be >= 0", what);
  *k = FtrlArgs{-(double)lr_power, lr, l1, 2.f * l2a, 2.f * l2_shrinkage, l2_shrinkage > 0.f ? 1 : 0};
  *mode = lr_power == -0.5f ? FT_SQRT : FT_POW;
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_sparse_ftrl_workspace_bytes(int64_t n) { return ag_group_workspace_bytes(n > 0 ? n : 1); }

extern "C" int tfrs_sparse_ftrl_f32(float* table, float* accum, float* linear, int64_t rows, int d, const void* ids,
                                    int ids_dtype, int64_t n, const float* grad_rows, float lr, float lr_power, float l1,
                                    float l2a, float l2_shrinkage, void* ws, size_t ws_bytes, void* stream) {
  int mode, rc;
  if ((rc = ag_check_args("sparse_ftrl", table && accum && linear, rows, d, ids_dtype, n, ids, grad_rows)) != TFRS_OK) return rc;
  TFRS_CHECK_ARG(d <= 1024, "sparse_ftrl: d=%d > 1024", d);
  FtrlArgs k;
  if ((rc = ft_args("sparse_ftrl", lr, lr_power, l1, l2a, l2_shrinkage, &k, &mode)) != TFRS_OK) return rc;
  if (n == 0) return TFRS_OK;
  if (!ws || ws_bytes < tfrs_sparse_ftrl_workspace_bytes(n)) {
    set_error("sparse_ftrl: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  AgGroups gr;
  if ((rc = ag_group(ids, ids_dtype, n, rows, ws, st, &gr)) != TFRS_OK) return rc;
  if (mode == FT_SQRT) return ag_run_sums(gr, n, grad_rows, d, FtrlRowOp<FT_SQRT>{table, accum, linear, k}, st);
  return ag_run_sums(gr, n, grad_rows, d, FtrlRowOp<FT_POW>{table, accum, linear, k}, st);
}

extern "C" int tfrs_ftrl_dense_f32(float* const* vars, const float* const* grads, float* const* accums,
                                   float* const* linears, const int64_t* numels, int nvars, float lr, float lr_power,
                                   float l1, float l2a, float l2_shrinkage, void* stream) {
  TFRS_CHECK_ARG(nvars >= 0, "ftrl_dense: nvars=%d < 0", nvars);
  FtrlArgs k;
  int mode, rc;
  if ((rc = ft_args("ftrl_dense", lr, lr_power, l1, l2a, l2_shrinkage, &k, &mode)) != TFRS_OK) return rc;
  if (nvars == 0) return TFRS_OK;
  TFRS_CHECK_ARG(vars && grads && accums && linears && numels, "ftrl_dense: NULL descriptor array");
  for (int i = 0; i < nvars; ++i) {
    TFRS_CHECK_ARG(numels[i] >= 0 && numels[i] < (1ll << 40), "ftrl_dense: numel[%d]=%lld out of range", i,
                   (long long)numels[i]);
    TFRS_CHECK_ARG(numels[i] == 0 || (vars[i] && grads[i] && accums[i] && linears[i]),
                   "ftrl_dense: NULL pointer for variable %d", i);
  }
  cudaStream_t st = (cudaStream_t)stream;
  return mt_for_each_batch<FtVar, FT_MAX>(
      nvars, numels, "ftrl_dense",
      [&](int i) { return FtVar{vars[i], grads[i], accums[i], linears[i], numels[i]}; },
      [&](const FtBatch& b, unsigned blocks, int) {
        if (mode == FT_SQRT) ft_dense_apply<FT_SQRT><<<blocks, MT_THREADS, 0, st>>>(b, k);
        else ft_dense_apply<FT_POW><<<blocks, MT_THREADS, 0, st>>>(b, k);
        TFRS_LAUNCH_CHECK();
        return TFRS_OK;
      });
}
