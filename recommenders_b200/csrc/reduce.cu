// reduce.cu -- the fixed-order reductions shared by the layers: the fp32 sum of split-K / chunk / part partials and the fp64
// sum of a loss vector or of each column of a row-major matrix.  The summation order is fixed, so every result is bitwise reproducible; there are no float atomics.
#include "common.cuh"

namespace tfrs {

// out[m*ld + n] = sum_z partial[z][m*N + n], z ascending, in fp32
__global__ void __launch_bounds__(256)
reduce_parts_kernel(const float* __restrict__ partial, long long M, long long N, int parts, float* __restrict__ out, long long ld) {
  const long long elems = M * N, e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e >= elems) return;
  float a = partial[e];
  for (int z = 1; z < parts; ++z) a += partial[(long long)z * elems + e];
  out[ld == N ? e : (e / N) * ld + e % N] = a;
}

int reduce_parts(const float* partial, long long M, long long N, int parts, float* out, long long ld, cudaStream_t st) {
  reduce_parts_kernel<<<(unsigned)ceil_div(M * N, 256), 256, 0, st>>>(partial, M, N, parts, out, ld);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// loss[c] = sum_i v[i * stride + c], i < n, c = blockIdx.x: fp64 per-thread sums (thread t takes i = t, t + 1024, ...),
// then a fixed tree
__global__ void __launch_bounds__(1024)
reduce_loss_kernel(const float* __restrict__ v, long long n, long long stride, float* __restrict__ loss) {
  __shared__ double red[1024];
  v += blockIdx.x;
  loss += blockIdx.x;
  double a = 0.0;
  for (long long i = threadIdx.x; i < n; i += 1024) a += (double)v[i * stride];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) { if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s]; __syncthreads(); }
  if (threadIdx.x == 0) loss[0] = (float)red[0];
}

int reduce_loss(const float* v, long long n, long long stride, float* loss, cudaStream_t st) {
  reduce_loss_kernel<<<1, 1024, 0, st>>>(v, n, stride, loss);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

int reduce_columns(const float* v, long long n, long long cols, float* out, cudaStream_t st) {
  reduce_loss_kernel<<<(unsigned)cols, 1024, 0, st>>>(v, n, cols, out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

}  // namespace tfrs
