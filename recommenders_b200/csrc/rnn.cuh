// rnn.cuh -- what the recurrence kernels K19 (gru.cu) and K20 (lstm.cu) share: the gate arithmetic, the plan of a
// CTA's (row, unit) pairs, the shared-memory budget and the choice of kernel instance.  Nothing here depends on the
// cell; each file brings its own kernels.  The gate derivatives are taken from the saved gate OUTPUTS, as TF's
// SigmoidGrad / TanhGrad do.
#pragma once
#include "dense.cuh"

namespace tfrs {

// 1 / (1 + expf(-x)): the Dense layer's sigmoid
__device__ __forceinline__ float rnn_sigmoid(float x) { return dense_act(TFRS_ACT_SIGMOID, x); }
__device__ __forceinline__ float rnn_tanh(float x) { return tanhf(x); }
// sigmoid'(x) = s (1 - s) and tanh'(x) = 1 - y^2 from s = sigmoid(x), y = tanh(x)
__device__ __forceinline__ float rnn_sigmoid_grad(float s) { return s * (1.f - s); }
__device__ __forceinline__ float rnn_tanh_grad(float y) { return 1.f - y * y; }

constexpr int RNN_THREADS = 256;
constexpr int RNN_PAIRS = 8;                  // (row, unit) pairs per thread: R * JT = RNN_THREADS * RNN_PAIRS / UJ
constexpr int RNN_SMEM_MAX = 227 * 1024;      // sm_90 opt-in dynamic shared memory per block
constexpr int RNN_SLICE_BYTES = 64 * 1024;    // a streamed slice of U (or U^T) when the whole matrix does not fit

// Thread (j0, g) of a CTA owns hidden units j = j0 + JT*a (a < UJ) of the tile rows g + G*i (i < RJ).
struct RnnTile {
  int jt, g, uj, rj, rows;
};

static inline RnnTile rnn_tile(int u) {
  RnnTile t;
  t.jt = 32;   // a power of two, so that the G = RNN_THREADS / JT row groups use every thread and no two alias a row
  while (t.jt < u && t.jt < RNN_THREADS) t.jt *= 2;
  t.g = RNN_THREADS / t.jt;
  t.uj = 1;    // a power of two too, so that RJ = RNN_PAIRS / UJ is exact and names a kernel instance (rnn_tiles)
  while (t.uj * t.jt < u) t.uj *= 2;
  t.rj = RNN_PAIRS / t.uj;
  t.rows = t.g * t.rj;
  return t;
}

// shared memory of one CTA: the fixed part plus a weight matrix of `rows_total` rows of `per` floats, whole when it
// fits in the 227 KB, otherwise in slices of RNN_SLICE_BYTES (*slice_rows rows)
static inline void rnn_smem(int fixed_floats, int rows_total, int per, int* slice_rows, size_t* bytes) {
  const size_t fixed = (size_t)fixed_floats * 4, whole = (size_t)rows_total * per * 4;
  if (fixed + whole <= (size_t)RNN_SMEM_MAX) {
    *slice_rows = rows_total;
    *bytes = fixed + whole;
    return;
  }
  int s = RNN_SLICE_BYTES / (per * 4);
  *slice_rows = s < 1 ? 1 : s;
  *bytes = fixed + (size_t)*slice_rows * per * 4;
}

// L<M, UJ, RJ>::run for the tile of u (UJ units per thread, RJ = RNN_PAIRS / UJ rows)
template <template <typename, int, int> class L, typename M, typename A>
static int rnn_tiles(const char* what, int uj, const A& a, unsigned grid, size_t smem, cudaStream_t st) {
  switch (uj) {
    case 1: return L<M, 1, 8>::run(a, grid, smem, st);
    case 2: return L<M, 2, 4>::run(a, grid, smem, st);
    case 4: return L<M, 4, 2>::run(a, grid, smem, st);
    case 8: return L<M, 8, 1>::run(a, grid, smem, st);
  }
  set_error("%s: no kernel instance for %d units per thread", what, uj);
  return TFRS_ERR_INVALID_ARG;
}

// ... and for the mask's element type
template <template <typename, int, int> class L, typename A>
static int rnn_dispatch(const char* what, int mask_kind, int uj, const A& a, unsigned grid, size_t smem,
                        cudaStream_t st) {
  return mask_dispatch(a.mask, mask_kind,
                       [&](auto m) { return rnn_tiles<L, decltype(m)>(what, uj, a, grid, smem, st); });
}

static inline int rnn_check(const char* what, int64_t B, int64_t T, int u, int max_units, const void* mask,
                            int mask_kind) {
  TFRS_CHECK_ARG(B >= 0 && B < (1ll << 31) && T >= 1 && T < (1ll << 31) && u >= 1 && u <= max_units,
                 "%s: bad shape B=%lld T=%lld units=%d (1 <= units <= %d, T >= 1)", what, (long long)B, (long long)T, u,
                 max_units);
  TFRS_CHECK_MASK(what, mask, mask_kind);
  return TFRS_OK;
}

}  // namespace tfrs
