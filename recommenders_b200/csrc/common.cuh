// common.cuh -- shared helpers for libtfrs_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/tfrs_b200.h"

namespace tfrs {

// thread-local error text behind tfrs_last_error()
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define TFRS_CHECK_ARG(cond, ...)                          \
  do {                                                     \
    if (!(cond)) {                                         \
      ::tfrs::set_error(__VA_ARGS__);                      \
      return TFRS_ERR_INVALID_ARG;                         \
    }                                                      \
  } while (0)

#define TFRS_CUDA(expr)                                                                          \
  do {                                                                                           \
    cudaError_t e__ = (expr);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      ::tfrs::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__));   \
      return TFRS_ERR_CUDA;                                                                      \
    }                                                                                            \
  } while (0)

#define TFRS_LAUNCH_CHECK()                                                                      \
  do {                                                                                           \
    ::tfrs::count_launch();                                                                      \
    cudaError_t e__ = cudaGetLastError();                                                        \
    if (e__ != cudaSuccess) {                                                                    \
      ::tfrs::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return TFRS_ERR_CUDA;                                                                      \
    }                                                                                            \
  } while (0)

// ---- Keras masks (include/tfrs_b200.h): kind TFRS_BOOL / TFRS_I32 / TFRS_I64, nonzero = kept, NULL keeps everything
#define TFRS_CHECK_MASK(what, mask, kind)                                                     \
  TFRS_CHECK_ARG(!(mask) || (kind) == TFRS_I32 || (kind) == TFRS_I64 || (kind) == TFRS_BOOL, \
                 "%s: a mask must be I32, I64 or BOOL", what)

// element i of a mask of element type M (uint8_t for BOOL, int32_t, long long), true for a NULL mask
template <typename M>
__device__ __forceinline__ bool mask_kept(const void* m, long long i) {
  return m == nullptr || static_cast<const M*>(m)[i] != 0;
}

// element i of a non-NULL mask of a runtime kind.  Callers test for NULL themselves: folding that test in here changes
// the code of the K21 and K25 kernels.
__device__ __forceinline__ bool mask_kept(const void* m, int kind, long long i) {
  if (kind == TFRS_BOOL) return static_cast<const uint8_t*>(m)[i] != 0;
  if (kind == TFRS_I32) return static_cast<const int32_t*>(m)[i] != 0;
  return static_cast<const long long*>(m)[i] != 0;
}

// f(M{}) with M the element type of a checked mask; no mask runs the uint8_t instance
template <typename F>
static int mask_dispatch(const void* mask, int kind, F f) {
  if (!mask || kind == TFRS_BOOL) return f(uint8_t{});
  if (kind == TFRS_I32) return f(int32_t{});
  return f((long long)0);
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// (score desc, index asc): the total order of tf.math.top_k that the whole path relies on.
__host__ __device__ __forceinline__ bool better(float sa, long long ia, float sb, long long ib) {
  return (sa > sb) || (sa == sb && ia < ib);
}

// |v| for the rescale statistic max |element|, 0 for Inf and NaN: one non-finite element makes only its own row or column
// of a split-fp16 product non-finite, instead of leaving the whole operand unscaled.  Every producer of that statistic
// (tc_split.cuh cx_amax_kernel, the CROSS epilogue's out_amax, cross.cu cross_bwd_elem) uses it, so they agree bit for bit.
__device__ __forceinline__ float finite_abs(float v) {
  const float a = fabsf(v);
  return a < INFINITY ? a : 0.f;
}

int sm_count();  // SMs of the CURRENT device (cached per device)

// 256-thread blocks for a grid-stride loop over n elements: one element per thread, at most 16 blocks per SM
static inline unsigned elementwise_grid(long long n) {
  const long long want = ceil_div(n, 256), cap = (long long)sm_count() * 16;
  return (unsigned)(want < cap ? want : cap);
}

// Fixed-order reductions (reduce.cu), one launch each.
// out[m*ld + n] = sum_z partial[z][m*N + n] over z = 0 .. parts-1 ascending, in fp32
int reduce_parts(const float* partial, long long M, long long N, int parts, float* out, long long ld, cudaStream_t st);
// loss[0] = sum_i v[i * stride] over i < n, in fp64 and a fixed order
int reduce_loss(const float* v, long long n, long long stride, float* loss, cudaStream_t st);
// out[c] = sum_i v[i * cols + c] over i < n, for each c < cols: one CTA per column, fp64, the order of reduce_loss
int reduce_columns(const float* v, long long n, long long cols, float* out, cudaStream_t st);

// Hook of the sharded scan (topk_tc.cu <-> comm.cu): all device pointers; thr[q] = L_q - margin_q in the shard's screening
// units (scores scaled by 2^(*exp_corpus + qexp[q])), cut[q] = 2 eps_q.  The hook may raise thr[].
typedef int (*ThrHook)(void* ctx, float* thr, const float* margin, const float* cut, const int* qexp, const int* exp_corpus,
                       long long Q, cudaStream_t st);
int tc_topk_sharded_local(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d, int k,
                          int64_t index_offset, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes, void* stream,
                          ThrHook hook, void* hook_ctx);

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (call site, device): function attributes belong to
// a device/context, so a process-wide "done" flag would leave the second GPU of a process at the 48 KB default.
struct DeviceOnce {
  unsigned char done_[64] = {};
  int dev_ = 0;
  bool need() { if (cudaGetDevice(&dev_) != cudaSuccess) dev_ = 0; dev_ &= 63; return __atomic_load_n(&done_[dev_], __ATOMIC_ACQUIRE) == 0; }
  void done() { __atomic_store_n(&done_[dev_], (unsigned char)1, __ATOMIC_RELEASE); }
};
#define TFRS_DYN_SMEM(kernel, bytes)                                                                              \
  do {                                                                                                            \
    static ::tfrs::DeviceOnce once__;                                                                             \
    if (once__.need()) {                                                                                          \
      TFRS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));         \
      /* without the carve-out hint the driver sizes the L1/shared split for ONE block of this kernel, which caps   \
         multi-block-per-SM kernels (the warp-per-query finalize) at one resident block */                          \
      TFRS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,                        \
                                     (int)cudaSharedmemCarveoutMaxShared));                                         \
      once__.done();                                                                                              \
    }                                                                                                             \
  } while (0)

}  // namespace tfrs
