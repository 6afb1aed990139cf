// bags.cuh -- the bag rules of ragged (values, row_splits) inputs, shared by K8 (unified_embedding.cu) and K11
// (embedding_bag.cu).  row_splits is int64 [n_bags + 1] over n values; the caller guarantees n_bags >= 1 wherever a value
// looks for its bag.
#pragma once
#include "common.cuh"

namespace tfrs {

// Bag b's values [*s0, *s1): its splits clamped to [0, n], the end to at least the start.
template <typename F>
__device__ __forceinline__ void bag_range(const F& f, long long b, long long* s0, long long* s1) {
  const long long a = min(max((long long)__ldg(f.splits + b), 0ll), f.n);
  *s0 = a;
  *s1 = min(max((long long)__ldg(f.splits + b + 1), a), f.n);
}

// The bag of value v: the last bag whose first value is <= v (binary search over bags 0 .. n_bags-1).  v may still lie
// outside that bag's bag_range.
template <typename F>
__device__ __forceinline__ long long bag_of(const F& f, long long v) {
  long long lo = 0, hi = f.n_bags;
  while (hi - lo > 1) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(f.splits + mid) <= v) lo = mid; else hi = mid;
  }
  return lo;
}

}  // namespace tfrs
