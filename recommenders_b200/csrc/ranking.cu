// ranking.cu -- the ranking task's loss and metrics (tasks/ranking.py:26-119 with the tf.keras losses / metrics of the
// tutorials: BinaryCrossentropy, MeanSquaredError, BinaryAccuracy, AUC, Mean of predictions / labels, (R)MSE).
//   rk_fwd_kernel: a CTA per 2048 predictions; per-example loss, the CTA's weighted loss sum and metric sums (fixed-order
//   tree in shared memory, float64) and the CTA's AUC bucket histograms (bucket b summed by one thread walking the CTA's
//   rows in order) -> one partial record per CTA.
//   rk_fold_kernel: record slot s summed over the CTAs in ascending order -> the loss scalar and the batch statistics.
//   No float atomics anywhere: the loss, the statistics and the AUC are bitwise reproducible.
#include "common.cuh"

namespace tfrs {

constexpr int RK_ROWS = 2048;    // predictions per CTA
constexpr int RK_THREADS = 256;
constexpr int RK_SUMS = 1 + TFRS_RANKING_STATS;   // weighted loss sum + the statistics
constexpr float RK_EPS = 1e-7f;  // tf.keras.backend.epsilon(), the clip of binary_crossentropy

struct RkArgs {
  const float* loss_in; const float* pred; const float* labels; const float* w;
  long long B; int kind; float* per_example; float threshold; int T; double* partial;
};

__device__ __forceinline__ float rk_loss(int kind, float x, float y) {
  if (kind == TFRS_LOSS_BCE) {           // tf.keras.backend.binary_crossentropy, from probabilities
    const float p = fminf(fmaxf(x, RK_EPS), 1.f - RK_EPS);
    return -(y * logf(p + RK_EPS) + (1.f - y) * logf(1.f - p + RK_EPS));
  }
  if (kind == TFRS_LOSS_BCE_LOGITS)      // tf.nn.sigmoid_cross_entropy_with_logits
    return fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
  const float d = x - y;
  return d * d;
}

__device__ __forceinline__ float rk_dloss(int kind, float x, float y) {
  if (kind == TFRS_LOSS_BCE) {           // clip_by_value passes no gradient outside [eps, 1 - eps]
    if (!(x >= RK_EPS && x <= 1.f - RK_EPS)) return 0.f;
    return -y / (x + RK_EPS) + (1.f - y) / (1.f - x + RK_EPS);
  }
  if (kind == TFRS_LOSS_BCE_LOGITS) return 1.f / (1.f + expf(-x)) - y;
  return 2.f * (x - y);
}

template <bool LOSS, bool STATS>
__global__ void __launch_bounds__(RK_THREADS)
rk_fwd_kernel(const RkArgs a) {
  __shared__ int s_bucket[RK_ROWS];
  __shared__ float s_w[RK_ROWS], s_y[RK_ROWS];
  __shared__ double red[RK_SUMS][RK_THREADS];
  const long long r0 = (long long)blockIdx.x * RK_ROWS;
  const int n = (int)(a.B - r0 < RK_ROWS ? a.B - r0 : RK_ROWS);
  const int tid = threadIdx.x;
  double s[RK_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int j = tid; j < n; j += RK_THREADS) {
    const long long r = r0 + j;
    const float y = a.labels[r], w = a.w ? a.w[r] : 1.f;
    if (LOSS) {
      const float wl = w * rk_loss(a.kind, a.loss_in[r], y);
      if (a.per_example) a.per_example[r] = wl;
      s[0] += (double)wl;
    }
    if (STATS) {
      const float p = a.pred[r];
      s[1] += (double)w;
      s[2] += ((p > a.threshold ? 1.f : 0.f) == y) ? (double)w : 0.0;   // binary_accuracy
      s[3] += (double)w * p;
      s[4] += (double)w * y;
      const double d = (double)p - (double)y;
      s[5] += (double)w * d * d;
      int b = (int)ceilf(p * (float)(a.T - 1)) - 1;     // tf-keras AUC, evenly spaced thresholds
      b = b < 0 ? 0 : (b > a.T - 1 ? a.T - 1 : b);
      s_bucket[j] = b; s_w[j] = w; s_y[j] = y;
    }
  }
#pragma unroll
  for (int q = 0; q < RK_SUMS; ++q) red[q][tid] = s[q];
  __syncthreads();
  for (int h = RK_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h) {
#pragma unroll
      for (int q = 0; q < RK_SUMS; ++q) red[q][tid] += red[q][tid + h];
    }
    __syncthreads();
  }
  double* rec = a.partial + (long long)blockIdx.x * (RK_SUMS + 2 * a.T);
  if (tid < RK_SUMS) rec[tid] = red[tid][0];
  if (STATS) {
    for (int b = tid; b < a.T; b += RK_THREADS) {
      double pos = 0.0, neg = 0.0;
      for (int j = 0; j < n; ++j) {
        if (s_bucket[j] == b) { pos += (double)s_w[j] * s_y[j]; neg += (double)s_w[j] * (1.f - s_y[j]); }
      }
      rec[RK_SUMS + b] = pos;
      rec[RK_SUMS + a.T + b] = neg;
    }
  }
}

// slot s of the records summed over the CTAs in order; slot 0 -> the loss, slots 1.. -> stats
__global__ void __launch_bounds__(256)
rk_fold_kernel(const double* __restrict__ partial, int blocks, int slots, long long B, int reduction, float* __restrict__ loss,
               double* __restrict__ stats) {
  const int s = blockIdx.x * 256 + threadIdx.x;
  if (s >= slots) return;
  double a = 0.0;
  for (int z = 0; z < blocks; ++z) a += partial[(long long)z * slots + s];
  if (s == 0) {
    if (loss) *loss = (float)(reduction == TFRS_REDUCTION_SUM_OVER_BATCH_SIZE ? (B > 0 ? a / (double)B : 0.0) : a);
  } else if (stats) {
    stats[s - 1] = a;
  }
}

__global__ void __launch_bounds__(256)
rk_bwd_kernel(const float* __restrict__ x, const float* __restrict__ labels, const float* __restrict__ w, long long B, int kind,
              int reduction, const float* __restrict__ grad, float* __restrict__ dx) {
  const long long r = (long long)blockIdx.x * 256 + threadIdx.x;
  if (r >= B) return;
  const float g = reduction == TFRS_REDUCTION_NONE ? grad[r] : grad[0];
  float v = g * (w ? w[r] : 1.f) * rk_dloss(kind, x[r], labels[r]);
  if (reduction == TFRS_REDUCTION_SUM_OVER_BATCH_SIZE) v = v / (float)B;
  dx[r] = v;
}

static int rk_blocks(long long B) { return (int)(B > 0 ? ceil_div(B, RK_ROWS) : 1); }

static int rk_run(const RkArgs& a0, bool loss_on, bool stats_on, int reduction, float* loss, double* stats, void* ws, size_t ws_bytes,
                  cudaStream_t st) {
  const int blocks = rk_blocks(a0.B);
  const int slots = RK_SUMS + 2 * a0.T;
  if (!ws || ws_bytes < (size_t)blocks * slots * 8) { set_error("ranking: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  RkArgs a = a0; a.partial = (double*)ws;
  if (a.B == 0) {   // empty batch: zero sums
    TFRS_CUDA(cudaMemsetAsync(ws, 0, (size_t)slots * 8, st));
  } else if (loss_on && stats_on) {
    rk_fwd_kernel<true, true><<<blocks, RK_THREADS, 0, st>>>(a);
  } else if (loss_on) {
    rk_fwd_kernel<true, false><<<blocks, RK_THREADS, 0, st>>>(a);
  } else {
    rk_fwd_kernel<false, true><<<blocks, RK_THREADS, 0, st>>>(a);
  }
  TFRS_LAUNCH_CHECK();
  rk_fold_kernel<<<(unsigned)ceil_div(slots, 256), 256, 0, st>>>(a.partial, a.B == 0 ? 1 : blocks, slots, a.B, reduction,
                                                                  loss_on ? loss : nullptr, stats_on ? stats : nullptr);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_ranking_workspace_bytes(int64_t B, int num_thresholds) {
  const int T = num_thresholds > 0 ? num_thresholds : 0;
  return align_up((size_t)rk_blocks(B) * (RK_SUMS + 2 * T) * 8, 256);
}

extern "C" int tfrs_ranking_loss_fwd_f32(const float* loss_in, const float* pred, const float* labels, const float* weights, int64_t B,
                                         int loss_kind, int reduction, float* per_example, float* loss, double* stats, float threshold,
                                         int num_thresholds, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(loss_in && labels, "ranking_loss_fwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0, "ranking_loss_fwd: bad batch size");
  TFRS_CHECK_ARG(loss_kind >= TFRS_LOSS_BCE && loss_kind <= TFRS_LOSS_MSE, "ranking_loss_fwd: unknown loss %d", loss_kind);
  TFRS_CHECK_ARG(reduction >= TFRS_REDUCTION_NONE && reduction <= TFRS_REDUCTION_SUM_OVER_BATCH_SIZE,
                 "ranking_loss_fwd: unknown reduction %d", reduction);
  TFRS_CHECK_ARG(reduction != TFRS_REDUCTION_NONE || per_example, "ranking_loss_fwd: reduction NONE needs per_example");
  TFRS_CHECK_ARG(reduction == TFRS_REDUCTION_NONE || loss, "ranking_loss_fwd: a reduced loss needs `loss`");
  TFRS_CHECK_ARG(!stats || (pred && num_thresholds > 1), "ranking_loss_fwd: statistics need pred and num_thresholds > 1");
  const RkArgs a{loss_in, pred, labels, weights, B, loss_kind, per_example, threshold, stats ? num_thresholds : 0, nullptr};
  return rk_run(a, true, stats != nullptr, reduction, loss, stats, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int tfrs_ranking_loss_bwd_f32(const float* loss_in, const float* labels, const float* weights, int64_t B, int loss_kind,
                                         int reduction, const float* grad, float* dloss_in, void* stream) {
  TFRS_CHECK_ARG(loss_in && labels && grad && dloss_in, "ranking_loss_bwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0, "ranking_loss_bwd: bad batch size");
  TFRS_CHECK_ARG(loss_kind >= TFRS_LOSS_BCE && loss_kind <= TFRS_LOSS_MSE, "ranking_loss_bwd: unknown loss %d", loss_kind);
  if (B == 0) return TFRS_OK;
  rk_bwd_kernel<<<(unsigned)ceil_div(B, 256), 256, 0, (cudaStream_t)stream>>>(loss_in, labels, weights, B, loss_kind, reduction, grad,
                                                                             dloss_in);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_ranking_metrics_f32(const float* pred, const float* labels, const float* weights, int64_t B, double* stats,
                                        float threshold, int num_thresholds, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(pred && labels && stats, "ranking_metrics: NULL pointer");
  TFRS_CHECK_ARG(B >= 0 && num_thresholds > 1, "ranking_metrics: bad batch size / num_thresholds");
  const RkArgs a{nullptr, pred, labels, weights, B, 0, nullptr, threshold, num_thresholds, nullptr};
  return rk_run(a, false, true, TFRS_REDUCTION_SUM, nullptr, stats, ws, ws_bytes, (cudaStream_t)stream);
}
