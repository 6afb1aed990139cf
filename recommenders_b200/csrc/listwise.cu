// listwise.cu -- K13: TF-Ranking's listwise losses (ListMLE, pairwise hinge, softmax) and NDCG on [B, L] lists.
//   lw_fwd_kernel: one warp per list, W = clamp(2048 / Lp, 1, 8) lists per CTA (Lp = L rounded up to a power of two).  The
//   warp stages its list's scaled scores and labels in shared memory, sorts with a bitonic sort in shared memory (labels
//   descending for ListMLE and the ideal NDCG ranking, predictions descending for the NDCG ranking), does its scans with warp
//   shuffles in fp64, and writes the per-list loss, dl/ds and the list's NDCG.  Each CTA writes one float64 record; the last
//   CTA to finish (an integer ticket, no float atomics) folds the records in a fixed order into the loss scalar and the NDCG
//   sums, so one kernel serves a call and every result is bitwise reproducible.
//   lw_bwd_kernel: dx = (g * dl/ds) * (1/T) + 0.
// The rules are written out in include/tfrs_b200.h (K13) and DESIGN.md §2 (A18).
#include "common.cuh"

namespace tfrs {

constexpr int LW_REC = 5;             // [sum w l, sum w ndcg, sum w, #lists with gain, #lists without gain]
constexpr int LW_CTA_ITEMS = 2048;    // staged items per CTA
constexpr unsigned LW_FULL = 0xffffffffu;

static int lw_pow2(int L) { int p = 1; while (p < L) p <<= 1; return p; }
static int lw_warps(int Lp) { const int w = LW_CTA_ITEMS / Lp; return w < 1 ? 1 : (w > 8 ? 8 : w); }
static size_t lw_smem(int W, int Lp) { return (size_t)W * Lp * (8 + 4 + 4 + 2); }

struct LwArgs {
  const float* pred; const float* labels; const float* w;
  long long B; int L, Lp, mode, reduction, topn;
  float inv_t; unsigned seed, call;
  float* per_list; float* dlds; float* ndcg; const float* disc;
  float* loss; double* ndcg_stats;
  double* rec; unsigned* counter;
};

__device__ __forceinline__ unsigned lw_fmix(unsigned h) {   // murmur3's 32-bit finalizer
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}

// ListMLE's tie key: fmix(fmix(fmix(fmix(seed) ^ call) ^ b) ^ i)
__device__ __forceinline__ unsigned lw_mix32(unsigned seed, unsigned call, unsigned b, unsigned i) {
  return lw_fmix(lw_fmix(lw_fmix(lw_fmix(seed) ^ call) ^ b) ^ i);
}

// a sort key that is smaller for a larger float (-0 is +0)
__device__ __forceinline__ unsigned lw_desc(float f) {
  const unsigned u = __float_as_uint(f == 0.f ? 0.f : f);
  return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}

// ascending bitonic sort of (key, idx) pairs by one warp; Lp is a power of two
__device__ void lw_sort(unsigned long long* key, unsigned short* ix, int Lp, int lane) {
  for (int k = 2; k <= Lp; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (Lp >> 1); t += 32) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), p = i + j;
        const unsigned long long ki = key[i], kp = key[p];
        const unsigned short ii = ix[i], ip = ix[p];
        const bool gt = ki > kp || (ki == kp && ii > ip);
        if (gt == ((i & k) == 0)) { key[i] = kp; key[p] = ki; ix[i] = ip; ix[p] = ii; }
      }
      __syncwarp();
    }
  }
}

__device__ __forceinline__ double lw_wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(LW_FULL, v, o);
  return v;
}

// sum of t over the lanes before (prefix) or after (suffix) this one
__device__ __forceinline__ double lw_excl_prefix(double t, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(LW_FULL, t, o); if (lane >= o) t += u; }
  const double e = __shfl_up_sync(LW_FULL, t, 1);
  return lane == 0 ? 0.0 : e;
}
__device__ __forceinline__ double lw_excl_suffix(double t, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_down_sync(LW_FULL, t, o); if (lane + o < 32) t += u; }
  const double e = __shfl_down_sync(LW_FULL, t, 1);
  return lane == 31 ? 0.0 : e;
}

// IDCG / DCG at the order in ix: sum over ranks r < min(topn, n) of (2^y - 1) * disc[r], sequential fp32 (lane 0)
__device__ float lw_dcg(const float* yv, const unsigned short* ix, const float* disc, int top) {
  float d = 0.f;
  for (int r = 0; r < top; ++r) d = __fadd_rn(d, __fmul_rn(exp2f(yv[ix[r]]) - 1.f, disc[r]));
  return d;
}

__global__ void __launch_bounds__(256, 2)
lw_fwd_kernel(const LwArgs a) {
  extern __shared__ __align__(16) unsigned char lw_sm[];
  __shared__ double s_rec[8][LW_REC];
  __shared__ double s_red[256];
  __shared__ bool s_last;
  const int W = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, Lp = a.Lp, L = a.L;
  unsigned long long* key = (unsigned long long*)lw_sm + (size_t)warp * Lp;
  double* dv = (double*)key;                       // after the sorts: the scan buffer
  float* sv = (float*)((unsigned long long*)lw_sm + (size_t)W * Lp) + (size_t)warp * Lp;
  float* yv = sv + (size_t)W * Lp;
  unsigned short* ix = (unsigned short*)(yv + (size_t)(W - warp) * Lp) + (size_t)warp * Lp;
  const long long b = (long long)blockIdx.x * W + warp;
  double r[LW_REC] = {0.0, 0.0, 0.0, 0.0, 0.0};

  if (b < a.B) {
    const float* pr = a.pred + b * L;
    const float* lb = a.labels + b * L;
    float* dl = a.dlds ? a.dlds + b * L : nullptr;
    const float wb = a.w ? a.w[b] : 1.f;
    const double wd = (double)wb;
    const bool ndcg_on = a.disc != nullptr;
    int nloc = 0;
    float mloc = -INFINITY;
    for (int i = lane; i < Lp; i += 32) {
      float y = -1.f, s = 0.f;
      if (i < L) {
        const float yl = lb[i];
        s = pr[i] * a.inv_t;
        if (yl >= 0.f) { y = yl == 0.f ? 0.f : yl; ++nloc; mloc = fmaxf(mloc, s); }
        else if (dl) dl[i] = 0.f;        // padding: no loss, no gradient
      }
      sv[i] = s; yv[i] = y;
    }
    const int n = __reduce_add_sync(LW_FULL, nloc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mloc = fmaxf(mloc, __shfl_xor_sync(LW_FULL, mloc, o));
    const double md = (double)mloc;
    const int top = a.topn < n ? a.topn : n;
    __syncwarp();

    // labels descending (ListMLE: ties by the hashed key), padding last
    float idcg = 0.f;
    if (a.mode == TFRS_LIST_LOSS_LISTMLE || ndcg_on) {
      for (int i = lane; i < Lp; i += 32) {
        const float y = yv[i];
        const unsigned lo = a.mode == TFRS_LIST_LOSS_LISTMLE ? lw_mix32(a.seed, a.call, (unsigned)b, (unsigned)i) : 0u;
        key[i] = y >= 0.f ? ((unsigned long long)lw_desc(y) << 32) | lo : ~0ull;
        ix[i] = (unsigned short)i;
      }
      __syncwarp();
      lw_sort(key, ix, Lp, lane);
      if (ndcg_on && lane == 0) idcg = lw_dcg(yv, ix, a.disc, top);
      __syncwarp();
    }

    double ld = 0.0;   // the list loss in fp64 (ListMLE, softmax)
    float lf = 0.f;    // the list loss in fp32
    if (a.mode == TFRS_LIST_LOSS_LISTMLE && n > 0) {
      // sorted positions k < n; lane owns [k0, k1).  S_k = sum_{j >= k} e_j, e_j = exp(s_pi(j) - m)
      const int c = (n + 31) >> 5, k0 = min(n, lane * c), k1 = min(n, k0 + c);
      double acc = 0.0;
      for (int k = k1 - 1; k >= k0; --k) { acc += exp((double)sv[ix[k]] - md); dv[k] = acc; }
      const double soff = lw_excl_suffix(acc, lane);
      double part = 0.0, pre = 0.0;
      for (int k = k0; k < k1; ++k) {
        const double S = dv[k] + soff;
        part += log(S) - ((double)sv[ix[k]] - md);
        pre += 1.0 / S;
        dv[k] = pre;
      }
      ld = lw_wsum(part);
      const double poff = lw_excl_prefix(pre, lane);
      for (int k = k0; k < k1; ++k) {   // dl/ds_pi(k) = e_k * sum_{j <= k} 1/S_j - 1
        const double g = exp((double)sv[ix[k]] - md) * (dv[k] + poff) - 1.0;
        if (dl) dl[ix[k]] = (float)(wd * g);
      }
      lf = (float)ld;
    } else if (a.mode == TFRS_LIST_LOSS_SOFTMAX && n > 0) {
      double S = 0.0, Y = 0.0, sy = 0.0;
      for (int i = lane; i < L; i += 32) {
        const float y = yv[i];
        if (y >= 0.f) { const double t = (double)sv[i] - md; S += exp(t); Y += (double)y; sy += (double)y * t; }
      }
      S = lw_wsum(S); Y = lw_wsum(Y); sy = lw_wsum(sy);
      ld = Y > 0.0 ? Y * log(S) - sy : 0.0;
      for (int i = lane; i < L; i += 32) {   // dl/ds_i = Y softmax_i - y_i
        const float y = yv[i];
        if (y >= 0.f && dl) {
          const double g = Y > 0.0 ? Y * exp((double)sv[i] - md) / S - (double)y : 0.0;
          dl[i] = (float)(wd * g);
        }
      }
      lf = (float)ld;
    } else if (a.mode == TFRS_LIST_LOSS_PAIRWISE_HINGE && n > 1) {
      // row i (lane-strided): r_i = sum_{j asc, y_i > y_j} max(0, 1 - (s_i - s_j)) in fp32; c_i = #active (j, i) - #active (i, j)
      float* rf = (float*)dv;
      int* rc = (int*)dv;
      int cloc = 0;
      for (int i = lane; i < L; i += 32) {
        const float yi = yv[i];
        if (!(yi >= 0.f)) continue;
        const float si = sv[i];
        float ri = 0.f;
        int ci = 0;
        for (int j = 0; j < L; ++j) {
          const float yj = yv[j];
          if (!(yj >= 0.f)) continue;
          if (yi > yj) {
            const float h = 1.f - (si - sv[j]);
            ri = ri + fmaxf(h, 0.f);
            ++cloc;
            if (h > 0.f) --ci;
          } else if (yj > yi) {
            if (1.f - (sv[j] - si) > 0.f) ++ci;
          }
        }
        rf[2 * i] = ri; rc[2 * i + 1] = ci;
      }
      const int cnt = __reduce_add_sync(LW_FULL, cloc);
      __syncwarp();
      if (lane == 0) {
        float sum = 0.f;
        for (int i = 0; i < L; ++i) if (yv[i] >= 0.f) sum = sum + rf[2 * i];
        lf = cnt > 0 ? sum / (float)cnt : 0.f;
      }
      lf = __shfl_sync(LW_FULL, lf, 0);
      for (int i = lane; i < L; i += 32) {
        if (yv[i] >= 0.f && dl) dl[i] = (float)(wd * (cnt > 0 ? (double)rc[2 * i + 1] / (double)cnt : 0.0));
      }
    } else if (a.mode != TFRS_LIST_LOSS_NONE && dl) {   // no valid item (or one, for the hinge): zero gradient
      for (int i = lane; i < L; i += 32) if (yv[i] >= 0.f) dl[i] = (float)(wd * 0.0);
    }
    const float wl = wb * lf;
    if (a.mode != TFRS_LIST_LOSS_NONE && a.per_list && lane == 0) a.per_list[b] = wl;
    r[0] = (double)wl;

    if (ndcg_on) {   // ranking by prediction descending, ties to the lower index
      __syncwarp();
      for (int i = lane; i < Lp; i += 32) {
        key[i] = yv[i] >= 0.f ? (unsigned long long)lw_desc(pr[i]) << 32 : ~0ull;
        ix[i] = (unsigned short)i;
      }
      __syncwarp();
      lw_sort(key, ix, Lp, lane);
      if (lane == 0) {
        const float dcg = lw_dcg(yv, ix, a.disc, top);
        const float nd = idcg > 0.f ? dcg / idcg : 0.f;
        if (a.ndcg) a.ndcg[b] = nd;
        if (idcg > 0.f) { r[1] = wd * (double)nd; r[2] = wd; r[3] = 1.0; }
        else r[4] = 1.0;
      }
    }
  }

  // per-CTA record: the warps' values summed in warp order
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < LW_REC; ++q) s_rec[warp][q] = r[q];
  }
  __syncthreads();
  if (threadIdx.x < LW_REC) {
    double v = 0.0;
    for (int w = 0; w < W; ++w) v += s_rec[w][threadIdx.x];
    a.rec[(size_t)blockIdx.x * LW_REC + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(a.counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();

  // the last CTA: slot q = tree over the threads of (thread t: records z = t, t + nt, ... ascending)
  const int nt = blockDim.x, t = threadIdx.x;
  double tot[LW_REC];
#pragma unroll
  for (int q = 0; q < LW_REC; ++q) {
    double v = 0.0;
    for (unsigned z = t; z < gridDim.x; z += nt) v += __ldcg(a.rec + (size_t)z * LW_REC + q);
    s_red[t] = v;
    __syncthreads();
    for (int h = nt >> 1; h > 0; h >>= 1) {
      if (t < h) s_red[t] += s_red[t + h];
      __syncthreads();
    }
    tot[q] = s_red[0];
    __syncthreads();
  }
  if (t == 0) {
    if (a.loss)
      *a.loss = (float)(a.reduction == TFRS_REDUCTION_SUM_OVER_BATCH_SIZE ? tot[0] / (double)a.B : tot[0]);
    if (a.ndcg_stats) {
      a.ndcg_stats[0] = tot[1];
      a.ndcg_stats[1] = __dadd_rn(tot[2], __dmul_rn(tot[4], tot[3] > 0.0 ? tot[2] / tot[3] : 0.0));   // no FMA
    }
  }
}

__global__ void __launch_bounds__(256)
lw_bwd_kernel(const float* __restrict__ dlds, long long B, int L, int reduction, float inv_t, const float* __restrict__ g,
              float* __restrict__ dx) {
  const long long n = B * L;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < n; e += (long long)gridDim.x * 256) {
    const float c = reduction == TFRS_REDUCTION_NONE ? g[e / L]
                  : (reduction == TFRS_REDUCTION_SUM_OVER_BATCH_SIZE ? g[0] / (float)B : g[0]);
    dx[e] = (c * dlds[e]) * inv_t + 0.f;   // + 0: a zero gradient (padding) is +0 whatever the sign of c
  }
}

static long long lw_blocks(long long B, int L) { return B > 0 ? ceil_div(B, lw_warps(lw_pow2(L))) : 0; }

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_listwise_workspace_bytes(int64_t B, int L) {
  if (B < 0 || L < 1 || L > TFRS_LISTWISE_MAX_LIST) return 0;
  return align_up((size_t)lw_blocks(B, L) * LW_REC * 8, 256) + 256;
}

extern "C" int tfrs_listwise_fwd_f32(const float* pred, const float* labels, const float* weights, int64_t B, int L, int loss_mode,
                                     int reduction, float inv_temperature, uint32_t seed, uint32_t call, float* per_list, float* loss,
                                     float* dlds, const float* discount, int topn, float* ndcg, double* ndcg_stats, void* ws,
                                     size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(pred && labels, "listwise_fwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0, "listwise_fwd: bad batch size");
  TFRS_CHECK_ARG(L >= 1 && L <= TFRS_LISTWISE_MAX_LIST, "listwise_fwd: list length %d outside [1, %d]", L, TFRS_LISTWISE_MAX_LIST);
  TFRS_CHECK_ARG(loss_mode >= TFRS_LIST_LOSS_NONE && loss_mode <= TFRS_LIST_LOSS_SOFTMAX, "listwise_fwd: unknown loss %d", loss_mode);
  TFRS_CHECK_ARG(reduction >= TFRS_REDUCTION_NONE && reduction <= TFRS_REDUCTION_SUM_OVER_BATCH_SIZE,
                 "listwise_fwd: unknown reduction %d", reduction);
  TFRS_CHECK_ARG(inv_temperature > 0.f && inv_temperature < INFINITY, "listwise_fwd: 1/temperature must be finite and > 0");
  TFRS_CHECK_ARG(loss_mode == TFRS_LIST_LOSS_NONE || reduction != TFRS_REDUCTION_NONE || per_list,
                 "listwise_fwd: reduction NONE needs per_list");
  TFRS_CHECK_ARG(loss_mode == TFRS_LIST_LOSS_NONE || reduction == TFRS_REDUCTION_NONE || loss, "listwise_fwd: a reduced loss needs `loss`");
  TFRS_CHECK_ARG(!(ndcg || ndcg_stats) || discount, "listwise_fwd: NDCG needs the discount table");
  TFRS_CHECK_ARG(loss_mode != TFRS_LIST_LOSS_NONE || ndcg || ndcg_stats, "listwise_fwd: nothing to compute");
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t need = tfrs_listwise_workspace_bytes(B, L);
  if (!ws || ws_bytes < need) { set_error("listwise_fwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  if (B == 0) {
    if (loss && loss_mode != TFRS_LIST_LOSS_NONE) TFRS_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
    if (ndcg_stats) TFRS_CUDA(cudaMemsetAsync(ndcg_stats, 0, 2 * sizeof(double), st));
    return TFRS_OK;
  }
  const int Lp = lw_pow2(L), W = lw_warps(Lp);
  const long long blocks = lw_blocks(B, L);
  TFRS_CHECK_ARG(blocks < (1ll << 31), "listwise_fwd: too many lists");
  unsigned* counter = (unsigned*)((char*)ws + need - 256);
  TFRS_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
  const bool with_ndcg = ndcg || ndcg_stats;
  const LwArgs a{pred, labels, weights, B, L, Lp, loss_mode, reduction, topn > 0 && topn < L ? topn : L, inv_temperature, seed, call,
                 loss_mode != TFRS_LIST_LOSS_NONE ? per_list : nullptr, loss_mode != TFRS_LIST_LOSS_NONE ? dlds : nullptr, ndcg,
                 with_ndcg ? discount : nullptr, loss_mode != TFRS_LIST_LOSS_NONE && reduction != TFRS_REDUCTION_NONE ? loss : nullptr,
                 ndcg_stats, (double*)ws, counter};
  lw_fwd_kernel<<<(unsigned)blocks, W * 32, lw_smem(W, Lp), st>>>(a);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_listwise_bwd_f32(const float* dlds, int64_t B, int L, int reduction, float inv_temperature, const float* grad,
                                     float* dx, void* stream) {
  TFRS_CHECK_ARG(dlds && grad && dx, "listwise_bwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0 && L >= 1 && L <= TFRS_LISTWISE_MAX_LIST, "listwise_bwd: bad shape");
  TFRS_CHECK_ARG(reduction >= TFRS_REDUCTION_NONE && reduction <= TFRS_REDUCTION_SUM_OVER_BATCH_SIZE,
                 "listwise_bwd: unknown reduction %d", reduction);
  if (B == 0) return TFRS_OK;
  lw_bwd_kernel<<<elementwise_grid(B * L), 256, 0, (cudaStream_t)stream>>>(dlds, B, L, reduction, inv_temperature, grad, dx);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
