// attention.cu -- K21: the attention core of tf.keras.layers.MultiHeadAttention (attention_axes over the sequence, no
// dropout).  The Q / K / V / output projections are K6 (dense.cu) and run around this file; here Q [B, T, H*dk], K [B, S,
// H*dk] and V [B, S, H*dv] are read in place (head h is columns h*dk .. h*dk + dk - 1 of a row), with no head transpose.
//
//   A team of MHA_LANES = 8 lanes owns one row of the side it iterates for: a query row (b, h, t) in the forward and the
//   dQ kernel, a key row (b, h, s) in the dK / dV kernel.  Lane l holds the head elements l + 8 i (i < E) of its row in
//   registers.  A CTA of 256 threads is 32 teams on 32 consecutive rows of the flat (b, h, row) order, so at short T a
//   CTA takes several (b, h) sequences (T = 10: up to 5) and every thread has a row.  The other side's rows of every
//   sequence the CTA touches are staged in shared memory, `tile` rows at a time, and all teams walk the same tile.
//   A score is the team's fmaf chains over i ascending, then a butterfly sum over the 8 lanes, so every lane holds it;
//   the three kernels compute it the same way, so the backward recomputes the forward's scores bit for bit.
//   forward: online softmax in fp32 (running max m and sum l, O rescaled when m grows), O = sum_j e^{s_j - m} v_j / l;
//     writes O, the row statistics (m, l) and, only when asked, P = e^{s - m} / l (a second walk over the keys).
//   backward: (1) delta = rowsum(dO * O); (2) per key row, over the query tiles: p = e^{s - m} / l, dV += p dO,
//     ds = p (dO.v - delta), dK += ds q; (3) per query row, over the key tiles: dq += ds k, dQ = dq * scale.  Every sum
//     runs in a fixed order: no atomics, bitwise reproducible.
//   l is in [1, S] (the max contributes e^0), so the divisions by l are __fdividef (2 ulp, no slow-path call).
//   Masks: a score the combined mask drops gets -1e9 added in fp32 (tf-keras Softmax), so a fully masked row is uniform.
#include "common.cuh"

namespace tfrs {

constexpr int MHA_THREADS = 256;
constexpr int MHA_LANES = 8;                              // lanes per row; a power of two dividing 32
constexpr int MHA_TEAMS = MHA_THREADS / MHA_LANES;        // rows per CTA
constexpr int MHA_MAX_TILE = 64;                          // staged rows per sequence
constexpr int MHA_SMEM_BUDGET = 64 * 1024;
constexpr float MHA_MASK_ADDER = -1e9f;                   // tf-keras _large_negative_number(float32)

struct MhaArgs {
  const float* q; const float* k; const float* v;
  const float* o; const float* dout; const float* stats; const float* delta;
  TfrsMhaMasks m; int masked;
  long long B; int T, S, H, dk, dv; float scale;
  int nseq, tile;                                         // sequences a CTA can touch; staged rows per sequence
  float* out; float* stats_out; float* p; float* dq; float* dk_out; float* dv_out; float* delta_out;
};

__device__ __forceinline__ bool mha_mask_at(const void* m, int kind, long long i) {
  if (kind == TFRS_BOOL) return static_cast<const uint8_t*>(m)[i] != 0;
  if (kind == TFRS_I32) return static_cast<const int32_t*>(m)[i] != 0;
  return static_cast<const long long*>(m)[i] != 0;
}

// score (b, t, s) kept by every mask present (tf-keras _compute_attention_mask: query & value & key & causal & attention)
__device__ __forceinline__ bool mha_keep(const MhaArgs& a, long long b, int t, int s) {
  const TfrsMhaMasks& m = a.m;
  if (m.query && !mha_mask_at(m.query, m.query_kind, b * a.T + t)) return false;
  if (m.value && !mha_mask_at(m.value, m.value_kind, b * a.S + s)) return false;
  if (m.key && !mha_mask_at(m.key, m.key_kind, b * a.S + s)) return false;
  if (m.causal && s > t) return false;
  if (m.attention && !mha_mask_at(m.attention, m.attention_kind, (b * a.T + t) * a.S + s)) return false;
  return true;
}

// the sum of x over the team's 8 lanes, in every lane (fixed butterfly order)
__device__ __forceinline__ float team_sum(float x) {
#pragma unroll
  for (int o = 1; o < MHA_LANES; o <<= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

template <int E>
__device__ __forceinline__ float team_dot(const float (&r)[E], const float* row, int n, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if (d < n) acc = fmaf(r[i], row[d], acc);
  }
  return team_sum(acc);
}

// The team's row: its flat index r over the rows of length L (T or S) of the B*H sequences; n = b*H + h, the row
// position w, and its slot among the sequences the CTA touches.  A team past the last row takes the CTA's first row
// r0 (always a real row), so every address it forms -- Q / K / V, dO, the row statistics, delta -- lies inside the
// caller's buffers, every lane of every warp reaches each shuffle, and `live` keeps it from writing.
struct MhaRow {
  int r, n, b, h, w, slot, nseq; bool live;
  __device__ MhaRow(int rows, int L, int H) {
    const int r0 = blockIdx.x * MHA_TEAMS;
    r = r0 + threadIdx.x / MHA_LANES;
    live = r < rows;
    if (!live) r = r0;
    const int n0 = r0 / L, last = (r0 + MHA_TEAMS < rows ? r0 + MHA_TEAMS : rows) - 1;
    n = r / L;
    w = r - n * L;
    b = n / H; h = n % H;
    slot = n - n0;
    nseq = last / L - n0 + 1;
  }
};

// rows j0 .. j0 + jn - 1 of head-row width `width` of every sequence n0 .. n0 + nseq - 1 into dst[slot][j][width];
// src row (b, j, h) is at src + ((b * L + j) * H + h) * width, scaled by `mul`
__device__ __forceinline__ void mha_stage(float* dst, const float* src, int n0, int nseq, int j0, int jn, int L, int H,
                                          int width, int tile, float mul) {
  const int total = nseq * jn * width;
  for (int e = threadIdx.x; e < total; e += MHA_THREADS) {
    const int d = e % width, rest = e / width;
    const int j = rest % jn, nn = n0 + rest / jn;
    const long long src_row = ((long long)(nn / H) * L + j0 + j) * H + nn % H;
    dst[((long long)(rest / jn) * tile + j) * width + d] = src[src_row * width + d] * mul;
  }
}

template <int E>
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_fwd_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const MhaRow row((int)(a.B * H * T), T, H);
  const int n0 = blockIdx.x * MHA_TEAMS / T;
  float* sK = sm;
  float* sV = sm + (size_t)a.nseq * a.tile * dk;

  float q[E], o[E];
  const long long qb = (((long long)row.b * T + row.w) * H + row.h) * (long long)dk;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    q[i] = d < dk ? a.q[qb + d] * a.scale : 0.f;     // Keras: query * (1 / sqrt(dk)) in fp32, then the scores
    o[i] = 0.f;
  }
  float mx = -INFINITY, l = 0.f;
  for (int s0 = 0; s0 < S; s0 += a.tile) {
    const int sn = min(a.tile, S - s0);
    __syncthreads();
    mha_stage(sK, a.k, n0, row.nseq, s0, sn, S, H, dk, a.tile, 1.f);
    mha_stage(sV, a.v, n0, row.nseq, s0, sn, S, H, dv, a.tile, 1.f);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    const float* vr = sV + (size_t)row.slot * a.tile * dv;
    for (int j = 0; j < sn; ++j) {
      float s = team_dot<E>(q, kr + j * dk, dk, lane);
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      if (s > mx) {
        const float c = expf(mx - s);
        l *= c;
#pragma unroll
        for (int i = 0; i < E; ++i) o[i] *= c;
        mx = s;
      }
      const float e = expf(s - mx);
      l += e;
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dv) o[i] = fmaf(e, vr[j * dv + d], o[i]);
      }
    }
  }
  if (row.live) {
    const long long ob = (((long long)row.b * T + row.w) * H + row.h) * (long long)dv;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const int d = lane + MHA_LANES * i;
      if (d < dv) a.out[ob + d] = __fdividef(o[i], l);
    }
    if (lane == 0 && a.stats_out) {
      a.stats_out[2ll * row.r] = mx;
      a.stats_out[2ll * row.r + 1] = l;
    }
  }
  if (!a.p) return;                                  // uniform: the whole CTA returns or none of it
  float* pr = a.p + (long long)row.r * S;                       // P [B, H, T, S]: row r = (b*H + h)*T + t
  for (int s0 = 0; s0 < S; s0 += a.tile) {
    const int sn = min(a.tile, S - s0);
    __syncthreads();
    mha_stage(sK, a.k, n0, row.nseq, s0, sn, S, H, dk, a.tile, 1.f);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    for (int j = 0; j < sn; ++j) {
      float s = team_dot<E>(q, kr + j * dk, dk, lane);
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      if (row.live && (j % MHA_LANES) == lane) pr[s0 + j] = __fdividef(expf(s - mx), l);
    }
  }
}

// delta[r] = sum_e dO[r, e] O[r, e] for the query rows r = (b*H + h)*T + t
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_delta_kernel(const MhaArgs a) {
  const int lane = threadIdx.x % MHA_LANES, T = a.T, H = a.H, dv = a.dv;
  const MhaRow row((int)(a.B * H * T), T, H);
  const long long ob = (((long long)row.b * T + row.w) * H + row.h) * (long long)dv;
  float acc = 0.f;
  if (row.live)
    for (int d = lane; d < dv; d += MHA_LANES) acc = fmaf(a.dout[ob + d], a.o[ob + d], acc);
  acc = team_sum(acc);
  if (row.live && lane == 0) a.delta_out[row.r] = acc;
}

// dK and dV of the key rows (b, h, s), walking the query rows of their sequence
template <int E>
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_bwd_kv_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const MhaRow row((int)(a.B * H * S), S, H);
  const int n0 = blockIdx.x * MHA_TEAMS / S;
  const size_t per = (size_t)a.nseq * a.tile;
  float* sQ = sm;
  float* sO = sQ + per * dk;
  float* sM = sO + per * dv;                         // [slot][j][2]: the row statistics (m, l)
  float* sD = sM + per * 2;                          // [slot][j]: delta

  float k[E], v[E], gk[E], gv[E];
  const long long kb = (((long long)row.b * S + row.w) * H + row.h) * (long long)dk;
  const long long vb = (((long long)row.b * S + row.w) * H + row.h) * (long long)dv;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    k[i] = d < dk ? a.k[kb + d] : 0.f;
    v[i] = d < dv ? a.v[vb + d] : 0.f;
    gk[i] = gv[i] = 0.f;
  }
  for (int t0 = 0; t0 < T; t0 += a.tile) {
    const int tn = min(a.tile, T - t0);
    __syncthreads();
    mha_stage(sQ, a.q, n0, row.nseq, t0, tn, T, H, dk, a.tile, a.scale);
    mha_stage(sO, a.dout, n0, row.nseq, t0, tn, T, H, dv, a.tile, 1.f);
    for (int e = threadIdx.x; e < row.nseq * tn; e += MHA_THREADS) {
      const int z = e / tn, j = e % tn;
      const long long qr = (long long)(n0 + z) * T + t0 + j;
      sM[((size_t)z * a.tile + j) * 2] = a.stats[2 * qr];
      sM[((size_t)z * a.tile + j) * 2 + 1] = a.stats[2 * qr + 1];
      sD[(size_t)z * a.tile + j] = a.delta[qr];
    }
    __syncthreads();
    const size_t base = (size_t)row.slot * a.tile;
    for (int j = 0; j < tn; ++j) {
      const float* qr = sQ + (base + j) * dk;
      const float* gr = sO + (base + j) * dv;
      float s = team_dot<E>(k, qr, dk, lane);
      if (a.masked && !mha_keep(a, row.b, t0 + j, row.w)) s += MHA_MASK_ADDER;
      const float p = __fdividef(expf(s - sM[(base + j) * 2]), sM[(base + j) * 2 + 1]);
      const float dp = team_dot<E>(v, gr, dv, lane);
      const float ds = p * (dp - sD[base + j]);
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dv) gv[i] = fmaf(p, gr[d], gv[i]);
        if (d < dk) gk[i] = fmaf(ds, qr[d], gk[i]);
      }
    }
  }
  if (!row.live) return;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if (d < dk) a.dk_out[kb + d] = gk[i];
    if (d < dv) a.dv_out[vb + d] = gv[i];
  }
}

// dQ of the query rows (b, h, t), walking the key rows of their sequence
template <int E>
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_bwd_q_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const MhaRow row((int)(a.B * H * T), T, H);
  const int n0 = blockIdx.x * MHA_TEAMS / T;
  float* sK = sm;
  float* sV = sm + (size_t)a.nseq * a.tile * dk;

  float q[E], g[E], gq[E];
  const long long qb = (((long long)row.b * T + row.w) * H + row.h) * (long long)dk;
  const long long ob = (((long long)row.b * T + row.w) * H + row.h) * (long long)dv;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    q[i] = d < dk ? a.q[qb + d] * a.scale : 0.f;
    g[i] = d < dv ? a.dout[ob + d] : 0.f;
    gq[i] = 0.f;
  }
  const float mx = a.stats[2ll * row.r], l = a.stats[2ll * row.r + 1], dl = a.delta[row.r];
  for (int s0 = 0; s0 < S; s0 += a.tile) {
    const int sn = min(a.tile, S - s0);
    __syncthreads();
    mha_stage(sK, a.k, n0, row.nseq, s0, sn, S, H, dk, a.tile, 1.f);
    mha_stage(sV, a.v, n0, row.nseq, s0, sn, S, H, dv, a.tile, 1.f);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    const float* vr = sV + (size_t)row.slot * a.tile * dv;
    for (int j = 0; j < sn; ++j) {
      float s = team_dot<E>(q, kr + j * dk, dk, lane);
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      const float p = __fdividef(expf(s - mx), l);
      const float ds = p * (team_dot<E>(g, vr + j * dv, dv, lane) - dl);
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dk) gq[i] = fmaf(ds, kr[j * dk + d], gq[i]);
      }
    }
  }
  if (!row.live) return;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if (d < dk) a.dq[qb + d] = gq[i] * a.scale;      // d(query * scale) / d query
  }
}

// The staged-tile plan: how many sequences 32 consecutive rows of length L can touch, and how many rows per sequence
// fit the shared-memory budget at `width` floats per staged row.
static void mha_plan(int L, int width, int* nseq, int* tile, size_t* smem) {
  const long long span = (MHA_TEAMS - 1 + L - 1) / L + 1;
  *nseq = (int)(span < MHA_TEAMS ? span : MHA_TEAMS);
  long long t = MHA_SMEM_BUDGET / ((long long)*nseq * width * 4);
  t = t < 1 ? 1 : (t > MHA_MAX_TILE ? MHA_MAX_TILE : t);
  *tile = (int)t;
  *smem = (size_t)*nseq * *tile * width * 4;
}

// head elements per lane: E * 8 >= max(dk, dv), E a power of two naming one kernel instance
static int mha_elems(int dk, int dv) {
  const int w = dk > dv ? dk : dv;
  int e = 1;
  while (e * MHA_LANES < w) e *= 2;
  return e;
}

enum { MHA_FWD, MHA_BWD_KV, MHA_BWD_Q };

// The opt-in shared-memory cap is set once per device and call site, so it is the plan's budget, which every plan fits
template <int E>
static int mha_launch_e(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  switch (which) {
    case MHA_FWD:
      TFRS_DYN_SMEM(mha_fwd_kernel<E>, MHA_SMEM_BUDGET);
      mha_fwd_kernel<E><<<grid, MHA_THREADS, smem, st>>>(a);
      break;
    case MHA_BWD_KV:
      TFRS_DYN_SMEM(mha_bwd_kv_kernel<E>, MHA_SMEM_BUDGET);
      mha_bwd_kv_kernel<E><<<grid, MHA_THREADS, smem, st>>>(a);
      break;
    default:
      TFRS_DYN_SMEM(mha_bwd_q_kernel<E>, MHA_SMEM_BUDGET);
      mha_bwd_q_kernel<E><<<grid, MHA_THREADS, smem, st>>>(a);
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

static int mha_launch(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  switch (mha_elems(a.dk, a.dv)) {
    case 1: return mha_launch_e<1>(which, a, grid, smem, st);
    case 2: return mha_launch_e<2>(which, a, grid, smem, st);
    case 4: return mha_launch_e<4>(which, a, grid, smem, st);
    case 8: return mha_launch_e<8>(which, a, grid, smem, st);
    case 16: return mha_launch_e<16>(which, a, grid, smem, st);
  }
  set_error("mha: no kernel instance for dk = %d, dv = %d", a.dk, a.dv);
  return TFRS_ERR_INVALID_ARG;
}

static int mha_check(const char* what, int64_t B, int64_t T, int64_t S, int H, int dk, int dv, const TfrsMhaMasks* m) {
  TFRS_CHECK_ARG(B >= 0 && T >= 1 && S >= 1 && H >= 1 && B < (1ll << 31) && T < (1ll << 31) && S < (1ll << 31) &&
                     B * H * (T > S ? T : S) < (1ll << 31),
                 "%s: bad shape B=%lld T=%lld S=%lld H=%d", what, (long long)B, (long long)T, (long long)S, H);
  TFRS_CHECK_ARG(dk >= 1 && dk <= TFRS_MHA_MAX_HEAD_DIM && dv >= 1 && dv <= TFRS_MHA_MAX_HEAD_DIM,
                 "%s: key_dim = %d and value_dim = %d must be in 1 .. %d", what, dk, dv, TFRS_MHA_MAX_HEAD_DIM);
  if (m) {
    const void* ps[4] = {m->query, m->value, m->key, m->attention};
    const int ks[4] = {m->query_kind, m->value_kind, m->key_kind, m->attention_kind};
    for (int i = 0; i < 4; ++i)
      TFRS_CHECK_ARG(!ps[i] || ks[i] == TFRS_I32 || ks[i] == TFRS_I64 || ks[i] == TFRS_BOOL,
                     "%s: a mask must be I32, I64 or BOOL", what);
  }
  return TFRS_OK;
}

static MhaArgs mha_args(const float* Q, const float* K, const float* V, const TfrsMhaMasks* masks, int64_t B, int64_t T,
                        int64_t S, int H, int dk, int dv) {
  MhaArgs a{};
  a.q = Q; a.k = K; a.v = V;
  if (masks) a.m = *masks;
  a.masked = a.m.query || a.m.value || a.m.key || a.m.attention || a.m.causal;
  a.B = B; a.T = (int)T; a.S = (int)S; a.H = H; a.dk = dk; a.dv = dv;
  a.scale = (float)(1.0 / sqrt((double)dk));
  return a;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_mha_fwd_f32(const float* Q, const float* K, const float* V, const TfrsMhaMasks* masks, int64_t B,
                                int64_t T, int64_t S, int H, int dk, int dv, float* O, float* stats, float* P,
                                void* stream) {
  int rc = mha_check("mha_fwd", B, T, S, H, dk, dv, masks);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(Q && K && V && O, "mha_fwd: NULL pointer");
  MhaArgs a = mha_args(Q, K, V, masks, B, T, S, H, dk, dv);
  a.out = O; a.stats_out = stats; a.p = P;
  size_t smem;
  mha_plan((int)T, dk + dv, &a.nseq, &a.tile, &smem);
  return mha_launch(MHA_FWD, a, (unsigned)ceil_div(B * H * T, MHA_TEAMS), smem, (cudaStream_t)stream);
}

extern "C" size_t tfrs_mha_bwd_workspace_bytes(int64_t B, int64_t T, int H) {
  const long long n = B > 0 && T > 0 && H > 0 ? B * T * H : 0;
  const size_t bytes = align_up((size_t)n * 4, 256);
  return bytes < 256 ? 256 : bytes;
}

extern "C" int tfrs_mha_bwd_f32(const float* Q, const float* K, const float* V, const TfrsMhaMasks* masks,
                                const float* O, const float* stats, const float* dO, int64_t B, int64_t T, int64_t S,
                                int H, int dk, int dv, float* dQ, float* dK, float* dV, void* ws, size_t ws_bytes,
                                void* stream) {
  int rc = mha_check("mha_bwd", B, T, S, H, dk, dv, masks);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(Q && K && V && O && stats && dO && dQ && dK && dV, "mha_bwd: NULL pointer");
  if (!ws || ws_bytes < tfrs_mha_bwd_workspace_bytes(B, T, H)) {
    set_error("mha_bwd: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "mha_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  MhaArgs a = mha_args(Q, K, V, masks, B, T, S, H, dk, dv);
  a.o = O; a.dout = dO; a.stats = stats; a.delta = static_cast<float*>(ws); a.delta_out = static_cast<float*>(ws);
  a.dq = dQ; a.dk_out = dK; a.dv_out = dV;
  const unsigned qgrid = (unsigned)ceil_div(B * H * T, MHA_TEAMS), kgrid = (unsigned)ceil_div(B * H * S, MHA_TEAMS);
  mha_delta_kernel<<<qgrid, MHA_THREADS, 0, st>>>(a);
  TFRS_LAUNCH_CHECK();
  size_t smem;
  mha_plan((int)S, dk + dv + 3, &a.nseq, &a.tile, &smem);   // key rows: the CTA's sequences follow S
  if ((rc = mha_launch(MHA_BWD_KV, a, kgrid, smem, st))) return rc;
  mha_plan((int)T, dk + dv, &a.nseq, &a.tile, &smem);
  return mha_launch(MHA_BWD_Q, a, qgrid, smem, st);
}
