// multi_tensor.cuh -- multi-tensor launches over a list of dense variables, shared by the dense ClippyAdagrad
// (clippy_adagrad.cu, K7) and the dense Adam (adam.cu, K10).  The per-variable descriptors go by value in the kernel
// parameters (__grid_constant__), up to MAX variables per launch; longer lists are split into several launches.  Each
// MT_THREADS-thread block owns MT_CHUNK consecutive elements of one variable:
//   v  = mt_find(b)                                      the block's variable (index into the batch)
//   e0 = mt_first(b, v)                                  its first element; thread t owns e0 + u * MT_THREADS, u < MT_PER_THREAD
// A kernel's parameters must stay under the 32764 bytes that CUDA 12.1+ allows on sm_90: each user static_asserts it on
// sizeof(MtBatch<Var, MAX>) plus its other parameters.
#pragma once
#include "common.cuh"

namespace tfrs {

constexpr int MT_THREADS = 256, MT_PER_THREAD = 4, MT_CHUNK = MT_THREADS * MT_PER_THREAD;

template <class Var, int MAX>
struct MtBatch {
  Var v[MAX];
  unsigned int block0[MAX + 1];   // first block of each variable; block0[nvars] = grid size
  int nvars;
};

template <class B>
__device__ __forceinline__ int mt_find(const B& b) {   // the variable of this block: last v with block0[v] <= blockIdx.x
  int lo = 0, hi = b.nvars - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (b.block0[mid] <= blockIdx.x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <class B>
__device__ __forceinline__ long long mt_first(const B& b, int v) {
  return (long long)(blockIdx.x - b.block0[v]) * MT_CHUNK + threadIdx.x;
}

// Splits variables 0 .. nvars-1 into batches of at most MAX variables and 2^31 - 1 blocks, in order, and calls
// launch(batch, blocks, v0) for every batch that has elements (v0 = the list index of the batch's first variable).
// make(i) returns the descriptor of variable i.  Returns the first error of launch, or TFRS_OK.
template <class Var, int MAX, class Make, class Launch>
int mt_for_each_batch(int nvars, const int64_t* numels, const char* what, Make make, Launch launch) {
  static thread_local MtBatch<Var, MAX> b;   // up to 32 KB: off the stack
  for (int v0 = 0; v0 < nvars;) {
    b.nvars = 0;
    long long blocks = 0;
    int v = v0;
    for (; v < nvars && b.nvars < MAX; ++v) {
      const long long nb = ceil_div(numels[v], MT_CHUNK);
      if (b.nvars > 0 && blocks + nb > 0x7FFFFFFFll) break;
      TFRS_CHECK_ARG(nb <= 0x7FFFFFFFll, "%s: variable %d too large", what, v);
      b.v[b.nvars] = make(v);
      b.block0[b.nvars] = (unsigned int)blocks;
      blocks += nb;
      ++b.nvars;
    }
    b.block0[b.nvars] = (unsigned int)blocks;
    if (blocks > 0) {
      const int rc = launch(b, (unsigned)blocks, v0);
      if (rc != TFRS_OK) return rc;
    }
    v0 = v;
  }
  return TFRS_OK;
}

}  // namespace tfrs
