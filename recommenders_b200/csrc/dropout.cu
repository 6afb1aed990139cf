// dropout.cu -- K23: tf.keras.layers.Dropout's training-mode output y = keep(m(i)) ? x[i] * scale : +0, one elementwise
// kernel for both directions (the backward is the same call on dy, the mask regenerated from the same key and call).
//   Mask element j (row-major in the noise shape) takes word j % 4 of Philox4x32-10 (philox.cuh) at counter
//   (g lo, g hi, call lo, call hi), g = j / 4, key (seed lo, seed hi); keep <=> (word >> 8) >= thr.
//   m(i) maps output element i to its mask element: the host drops size-1 axes, merges adjacent axes that share a
//   broadcast flag, and passes the merged sizes with the mask strides (0 along a broadcast axis).
//   Without broadcasting m(i) = i, and one thread takes the four elements of one Philox call (float4 when x and y are
//   16-byte aligned); with broadcasting one thread takes one element.  One launch.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace tfrs {

constexpr int DROP_THREADS = 256;

struct DropoutMap {
  int rank;               // merged axes, 1..4
  long long size[4];      // merged axis sizes, row-major
  long long mstride[4];   // mask-index stride of each merged axis; 0 along a broadcast axis
};

__device__ __forceinline__ float drop1(float v, uint32_t word, uint32_t thr, float scale) {
  return (word >> 8) >= thr ? v * scale : 0.f;
}

__device__ __forceinline__ uint32_t word_of(const uint4& r, int e) {
  return e == 0 ? r.x : e == 1 ? r.y : e == 2 ? r.z : r.w;
}

__global__ void __launch_bounds__(DROP_THREADS)
dropout_dense_kernel(const float* __restrict__ x, long long n, uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1,
                     uint32_t thr, float scale, int vec, float* __restrict__ y) {
  const long long groups = (n + 3) >> 2, stride = (long long)gridDim.x * DROP_THREADS;
  for (long long g = (long long)blockIdx.x * DROP_THREADS + threadIdx.x; g < groups; g += stride) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), c0, c1), k0, k1);
    const long long i = g << 2;
    if (vec && i + 3 < n) {
      const float4 v = reinterpret_cast<const float4*>(x)[g];
      reinterpret_cast<float4*>(y)[g] = make_float4(drop1(v.x, r.x, thr, scale), drop1(v.y, r.y, thr, scale),
                                                    drop1(v.z, r.z, thr, scale), drop1(v.w, r.w, thr, scale));
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (i + e < n) y[i + e] = drop1(x[i + e], word_of(r, e), thr, scale);
    }
  }
}

__global__ void __launch_bounds__(DROP_THREADS)
dropout_bcast_kernel(const float* __restrict__ x, long long n, DropoutMap map, uint32_t k0, uint32_t k1, uint32_t c0,
                     uint32_t c1, uint32_t thr, float scale, float* __restrict__ y) {
  const long long stride = (long long)gridDim.x * DROP_THREADS;
  for (long long i = (long long)blockIdx.x * DROP_THREADS + threadIdx.x; i < n; i += stride) {
    long long rem = i, m = 0;
#pragma unroll
    for (int a = 3; a >= 0; --a)
      if (a < map.rank) {
        const long long q = rem / map.size[a];
        m += (rem - q * map.size[a]) * map.mstride[a];
        rem = q;
      }
    const long long g = m >> 2;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), c0, c1), k0, k1);
    y[i] = drop1(x[i], word_of(r, (int)(m & 3)), thr, scale);
  }
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_dropout_f32(const float* x, int rank, const int64_t* shape, const int64_t* noise_shape, double rate,
                                uint64_t seed, uint64_t call, float* y, void* stream) {
  if (rank < 1 || rank > TFRS_DROPOUT_MAX_RANK) {
    set_error("dropout: rank %d is not supported (1 to %d)", rank, TFRS_DROPOUT_MAX_RANK);
    return TFRS_ERR_UNSUPPORTED;
  }
  TFRS_CHECK_ARG(shape, "dropout: NULL shape");
  TFRS_CHECK_ARG(rate >= 0.0 && rate < 1.0, "dropout: rate must be in [0, 1), got %g", rate);
  long long n = 1;
  for (int a = 0; a < rank; ++a) {
    TFRS_CHECK_ARG(shape[a] >= 0, "dropout: negative size %lld on axis %d", (long long)shape[a], a);
    TFRS_CHECK_ARG(!noise_shape || noise_shape[a] == shape[a] || noise_shape[a] == 1,
                   "dropout: noise_shape[%d] = %lld must be 1 or the input's %lld", a, (long long)noise_shape[a],
                   (long long)shape[a]);
    n *= shape[a];
  }
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && y, "dropout: NULL pointer");
  const uint32_t thr = (uint32_t)ceil(rate * 16777216.0);
  const float scale = (float)(1.0 / (1.0 - rate));
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32), c0 = (uint32_t)call, c1 = (uint32_t)(call >> 32);
  // merge the axes: size-1 axes drop out, adjacent axes with the same broadcast flag become one
  DropoutMap map = {};
  int bcast[4] = {0, 0, 0, 0}, r = 0;
  for (int a = 0; a < rank; ++a) {
    if (shape[a] == 1) continue;
    const int b = noise_shape && noise_shape[a] == 1;
    if (r > 0 && bcast[r - 1] == b) {
      map.size[r - 1] *= shape[a];
    } else {
      map.size[r] = shape[a];
      bcast[r++] = b;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (r == 0 || (r == 1 && !bcast[0])) {
    const int vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
    dropout_dense_kernel<<<elementwise_grid(ceil_div(n, 4)), DROP_THREADS, 0, st>>>(x, n, k0, k1, c0, c1, thr, scale,
                                                                                   vec, y);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  map.rank = r;
  long long s = 1;
  for (int a = r - 1; a >= 0; --a) {
    map.mstride[a] = bcast[a] ? 0 : s;
    if (!bcast[a]) s *= map.size[a];
  }
  dropout_bcast_kernel<<<elementwise_grid(n), DROP_THREADS, 0, st>>>(x, n, map, k0, k1, c0, c1, thr, scale, y);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
