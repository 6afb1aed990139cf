// attention.cuh -- the team-per-row attention kernels of K21 (attention.cu) and K25 (additive_attention.cu).  One kernel
// body per pass, instantiated per score mode:
//   K21_MHA   tf.keras.layers.MultiHeadAttention's core: s = (q * 1/sqrt(dk)) . k, every mask in the softmax.
//   K21_DOT   tf.keras.layers.Attention(score_mode="dot"): s = scale (q . k) with the learnable scale read from a device
//             pointer; the value and causal masks in the softmax, the query mask on the output; fused weight dropout.
//   K25_TANH  tf.keras.layers.Attention(score_mode="concat") and AdditiveAttention: s = wc * sum_d w_d tanhf(c (q_d +
//             k_d)), recomputed in the backward (no [B, Tq, Tv, d] tensor); masks and dropout as K21_DOT.
// The dense layers run as one head (H = 1) over the B * Tq query rows.
//
//   A team of MHA_LANES = 8 lanes owns one row of the side it iterates for: a query row (b, h, t) in the forward and the
//   dQ kernel, a key row (b, h, s) in the dK / dV kernel.  Lane l holds the head elements l + 8 i (i < E) of its row in
//   registers.  A CTA of 256 threads is 32 teams on 32 consecutive rows of the flat (b, h, row) order, so at short T a
//   CTA takes several (b, h) sequences (T = 10: up to 5) and every thread has a row.  The other side's rows of every
//   sequence the CTA touches are staged in shared memory, `tile` rows at a time, and all teams walk the same tile.
//   A score is the team's fmaf chains over i ascending, then a butterfly sum over the 8 lanes, so every lane holds it;
//   the three kernels compute it the same way, so the backward recomputes the forward's scores bit for bit.
//   forward: online softmax in fp32 (running max m and sum l, O rescaled when m grows), O = sum_j e^{s_j - m} z_j v_j / l;
//     writes O, the row statistics (m, l) and, only when asked, P = e^{s - m} z / l (a second walk over the keys).
//   backward: (1) delta = rowsum(dO * O); (2) per key row, over the query tiles: p = e^{s - m} / l, dV += p z dO,
//     ds = p (z dO.v - delta), dK += ds dS/dk; (3) per query row, over the key tiles: dq += ds dS/dq, and the per-row
//     partials of the score weights' gradients; the dense modes' dQ kernel takes z dO.v - delta as dO.(z v - O).  Every
//     sum runs in a fixed order: no atomics, bitwise reproducible.
//   z is the dropout factor of a weight: 1 without dropout, else keep ? 1 / (1 - rate) : 0, keep from Philox4x32-10 at
//   element e = (b Tq + t) Tv + s (K23's rule over the [B, Tq, Tv] weights).  Each staged tile's keep bytes are drawn
//   once per CTA into shared memory, one Philox call per four weights.
//   l is in [1, S] (the max contributes e^0), so the divisions by l are __fdividef (2 ulp, no slow-path call).
//   Masks: a score the softmax mask drops gets -1e9 added in fp32 (tf-keras), so a fully masked row is uniform.
#pragma once
#include "common.cuh"
#include "philox.cuh"

namespace tfrs {

constexpr int MHA_THREADS = 256;
constexpr int MHA_LANES = 8;                              // lanes per row; a power of two dividing 32
constexpr int MHA_TEAMS = MHA_THREADS / MHA_LANES;        // rows per CTA
constexpr int MHA_MAX_TILE = 64;                          // staged rows per sequence
constexpr int MHA_SMEM_BUDGET = 64 * 1024;
constexpr int MHA_KEEP_BYTES = MHA_TEAMS * MHA_MAX_TILE;  // the dense modes' keep bytes [team][tile], past the budget
constexpr float MHA_MASK_ADDER = -1e9f;                   // tf-keras _large_negative_number(float32)

enum { K21_MHA, K21_DOT, K25_TANH };

struct MhaArgs {
  const float* q; const float* k; const float* v;
  const float* o; const float* dout; const float* stats; const float* delta;
  TfrsMhaMasks m; int masked;
  long long B; int T, S, H, dk, dv; float scale;
  int nseq, tile;                                         // sequences a CTA can touch; staged rows per sequence
  float* out; float* stats_out; float* p; float* dq; float* dk_out; float* dv_out; float* delta_out;
  // the dense modes (H = 1)
  const float* score_scale;                               // dot / concat: [1], additive: [dk]; NULL = 1
  const float* concat_weight;                             // concat: [1]; NULL = 1
  int additive;                                           // K25: per-d weights (additive) or one scale inside tanh
  const void* omask; int omask_kind;                      // query mask [B, T]: zeroes output rows
  int drop; uint32_t thr, k0, k1, c0, c1; float drop_scale;
  float* part;                                            // per query row: the score weights' gradient partials
};

// score (b, t, s) kept by every mask present (tf-keras _compute_attention_mask: query & value & key & causal & attention)
__device__ __forceinline__ bool mha_keep(const MhaArgs& a, long long b, int t, int s) {
  const TfrsMhaMasks& m = a.m;
  if (m.query && !mask_kept(m.query, m.query_kind, b * a.T + t)) return false;
  if (m.value && !mask_kept(m.value, m.value_kind, b * a.S + s)) return false;
  if (m.key && !mask_kept(m.key, m.key_kind, b * a.S + s)) return false;
  if (m.causal && s > t) return false;
  if (m.attention && !mask_kept(m.attention, m.attention_kind, (b * a.T + t) * a.S + s)) return false;
  return true;
}

// the dense modes: query row r = b * T + t keeps its output
__device__ __forceinline__ bool dense_out_kept(const MhaArgs& a, long long r) {
  return !a.omask || mask_kept(a.omask, a.omask_kind, r);
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

// The score's unweighted part: q . k (dot modes, q already scaled), or sum_d w_d tanhf(c (q_d + k_d)) with the tanh of
// each of the lane's elements left in t (K25; the caller multiplies by wc)
template <int E, int MODE>
__device__ __forceinline__ float mha_score(const float (&r)[E], const float* row, int n, int lane, const float (&w)[E],
                                           float c, float (&t)[E]) {
  if constexpr (MODE != K25_TANH) {
    return team_dot<E>(r, row, n, lane);
  } else {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const int d = lane + MHA_LANES * i;
      t[i] = 0.f;
      if (d < n) {
        t[i] = tanhf(c * (r[i] + row[d]));
        acc = fmaf(w[i], t[i], acc);
      }
    }
    return team_sum(acc);
  }
}

// The score weights of the dense modes, read once per thread from device memory (no host sync): the multiplier of q
// (dot), and w_d, c and wc of K25
template <int E, int MODE>
__device__ __forceinline__ void dense_weights(const MhaArgs& a, int lane, float& mul, float (&w)[E], float& c,
                                              float& wc) {
  mul = a.scale;
  c = wc = 1.f;
#pragma unroll
  for (int i = 0; i < E; ++i) w[i] = 1.f;
  if constexpr (MODE == K21_DOT) {
    if (a.score_scale) mul *= *a.score_scale;
  } else if constexpr (MODE == K25_TANH) {
    if (a.concat_weight) wc = *a.concat_weight;
    if (a.score_scale && a.additive) {
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        w[i] = d < a.dk ? a.score_scale[d] : 0.f;
      }
    } else if (a.score_scale) {
      c = *a.score_scale;
    }
  }
}

__device__ __forceinline__ uint8_t dense_keep_word(const MhaArgs& a, const uint4& w, int k) {
  const uint32_t x = k == 0 ? w.x : k == 1 ? w.y : k == 2 ? w.z : w.w;
  return (x >> 8) >= a.thr;
}

__device__ __forceinline__ uint4 dense_philox(const MhaArgs& a, long long g) {
  return philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), a.c0, a.c1), a.k0, a.k1);
}

// Keep bytes z[team][j] of the CTA's query rows r0 + team (forward, dQ) against the staged key rows s0 .. s0 + sn - 1:
// the elements of one row are contiguous, so one work item is one Philox group of four.  Rows past the last are 0.
__device__ __forceinline__ void dense_keep_query_rows(uint8_t* z, const MhaArgs& a, int rows, int s0, int sn) {
  const int r0 = blockIdx.x * MHA_TEAMS, per = (a.tile + 3) / 4 + 1;   // groups sn <= tile elements can touch
  for (int it = threadIdx.x; it < MHA_TEAMS * per; it += MHA_THREADS) {
    const int team = it / per, gi = it - team * per, r = r0 + team;
    if (r >= rows) {
      if (gi == 0)
        for (int j = 0; j < sn; ++j) z[team * a.tile + j] = 0;
      continue;
    }
    const long long e0 = (long long)r * a.S + s0, g = (e0 >> 2) + gi;
    if (g > ((e0 + sn - 1) >> 2)) continue;
    const uint4 w = dense_philox(a, g);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long j = 4 * g + k - e0;
      if (j >= 0 && j < sn) z[team * a.tile + j] = dense_keep_word(a, w, k);
    }
  }
}

// Keep bytes z[team][j] of the CTA's key rows r0 + team (dK / dV) against the staged query rows t0 .. t0 + tn - 1 of
// their sequences: element (b T + t) S + s is contiguous over the CTA's key rows of one sequence, so the first team of
// each Philox group in that run draws the four words and writes its successors' bytes.  Rows past the last are 0.
__device__ __forceinline__ void dense_keep_key_rows(uint8_t* z, const MhaArgs& a, int rows, int t0, int tn) {
  const int r0 = blockIdx.x * MHA_TEAMS;
  for (int it = threadIdx.x; it < MHA_TEAMS * tn; it += MHA_THREADS) {
    const int team = it % MHA_TEAMS, j = it / MHA_TEAMS, r = r0 + team;
    if (r >= rows) {
      z[team * a.tile + j] = 0;
      continue;
    }
    const int b = r / a.S, s = r - b * a.S;
    const long long e = ((long long)b * a.T + t0 + j) * a.S + s;
    if (team > 0 && s > 0 && (e & 3) != 0) continue;      // a predecessor in this sequence draws this group
    const uint4 w = dense_philox(a, e >> 2);
    for (int k = (int)(e & 3), u = team; k < 4 && u < MHA_TEAMS && r0 + u < rows && s + (u - team) < a.S; ++k, ++u)
      z[u * a.tile + j] = dense_keep_word(a, w, k);
  }
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

template <int E, int MODE>
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_fwd_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const int rows = (int)(a.B * H * T);
  const MhaRow row(rows, T, H);
  const int n0 = blockIdx.x * MHA_TEAMS / T;
  float* sK = sm;
  float* sV = sm + (size_t)a.nseq * a.tile * dk;
  uint8_t* sZ = reinterpret_cast<uint8_t*>(sV + (size_t)a.nseq * a.tile * dv);
  const uint8_t* zr = sZ + (threadIdx.x / MHA_LANES) * a.tile;
  const bool drop = MODE != K21_MHA && a.drop;

  float q[E], o[E], w[E], t[E], mul, c, wc;
  dense_weights<E, MODE>(a, lane, mul, w, c, wc);
  const long long qb = (((long long)row.b * T + row.w) * H + row.h) * (long long)dk;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if constexpr (MODE != K21_MHA) q[i] = d < dk ? a.q[qb + d] : 0.f;
    else q[i] = d < dk ? a.q[qb + d] * mul : 0.f;   // Keras's MHA: query * (1 / sqrt(dk)) in fp32, then the scores
    o[i] = 0.f;
  }
  float mx = -INFINITY, l = 0.f;
  for (int s0 = 0; s0 < S; s0 += a.tile) {
    const int sn = min(a.tile, S - s0);
    __syncthreads();
    mha_stage(sK, a.k, n0, row.nseq, s0, sn, S, H, dk, a.tile, 1.f);
    mha_stage(sV, a.v, n0, row.nseq, s0, sn, S, H, dv, a.tile, 1.f);
    if (drop) dense_keep_query_rows(sZ, a, rows, s0, sn);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    const float* vr = sV + (size_t)row.slot * a.tile * dv;
    for (int j = 0; j < sn; ++j) {
      float s = mha_score<E, MODE>(q, kr + j * dk, dk, lane, w, c, t);
      if constexpr (MODE != K21_MHA) s *= MODE == K21_DOT ? mul : wc;
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      if (s > mx) {
        const float cf = expf(mx - s);
        l *= cf;
#pragma unroll
        for (int i = 0; i < E; ++i) o[i] *= cf;
        mx = s;
      }
      float e = expf(s - mx);
      l += e;
      if (drop) e = zr[j] ? e * a.drop_scale : 0.f;   // dropout scales the weights O sums, not the normaliser
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dv) o[i] = fmaf(e, vr[j * dv + d], o[i]);
      }
    }
  }
  if (row.live) {
    const long long ob = (((long long)row.b * T + row.w) * H + row.h) * (long long)dv;
    bool kept = true;
    if constexpr (MODE != K21_MHA) kept = dense_out_kept(a, row.r);
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const int d = lane + MHA_LANES * i;
      if (d < dv) a.out[ob + d] = kept ? __fdividef(o[i], l) : 0.f;
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
    if (drop) dense_keep_query_rows(sZ, a, rows, s0, sn);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    for (int j = 0; j < sn; ++j) {
      float s = mha_score<E, MODE>(q, kr + j * dk, dk, lane, w, c, t);
      if constexpr (MODE != K21_MHA) s *= MODE == K21_DOT ? mul : wc;
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      if (row.live && (j % MHA_LANES) == lane) {
        const float p = __fdividef(expf(s - mx), l);
        pr[s0 + j] = drop ? (zr[j] ? p * a.drop_scale : 0.f) : p;
      }
    }
  }
}

// delta[r] = sum_e dO[r, e] O[r, e] for the query rows r = (b*H + h)*T + t
static __global__ void __launch_bounds__(MHA_THREADS, 1)
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
template <int E, int MODE>
__global__ void __launch_bounds__(MHA_THREADS, 1)
mha_bwd_kv_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const int rows = (int)(a.B * H * S);
  const MhaRow row(rows, S, H);
  const int n0 = blockIdx.x * MHA_TEAMS / S;
  const size_t per = (size_t)a.nseq * a.tile;
  float* sQ = sm;
  float* sO = sQ + per * dk;
  float* sM = sO + per * dv;                         // [slot][j][2]: the row statistics (m, l)
  float* sD = sM + per * 2;                          // [slot][j]: delta
  uint8_t* sZ = reinterpret_cast<uint8_t*>(sD + per);
  const uint8_t* zr = sZ + (threadIdx.x / MHA_LANES) * a.tile;
  const bool drop = MODE != K21_MHA && a.drop;

  float k[E], v[E], gk[E], gv[E], w[E], t[E], mul, c, wc;
  dense_weights<E, MODE>(a, lane, mul, w, c, wc);
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
    mha_stage(sQ, a.q, n0, row.nseq, t0, tn, T, H, dk, a.tile, MODE == K21_MHA ? mul : 1.f);
    mha_stage(sO, a.dout, n0, row.nseq, t0, tn, T, H, dv, a.tile, 1.f);
    for (int e = threadIdx.x; e < row.nseq * tn; e += MHA_THREADS) {
      const int z = e / tn, j = e % tn;
      const long long qr = (long long)(n0 + z) * T + t0 + j;
      float m = a.stats[2 * qr];
      if constexpr (MODE != K21_MHA)
        if (!dense_out_kept(a, qr)) m = INFINITY;    // an output-masked query row: p = e^{s - inf} = 0, no gradient
      sM[((size_t)z * a.tile + j) * 2] = m;
      sM[((size_t)z * a.tile + j) * 2 + 1] = a.stats[2 * qr + 1];
      sD[(size_t)z * a.tile + j] = a.delta[qr];
    }
    if (drop) dense_keep_key_rows(sZ, a, rows, t0, tn);
    __syncthreads();
    const size_t base = (size_t)row.slot * a.tile;
    for (int j = 0; j < tn; ++j) {
      const float* qr = sQ + (base + j) * dk;
      const float* gr = sO + (base + j) * dv;
      float s = mha_score<E, MODE>(k, qr, dk, lane, w, c, t);
      if constexpr (MODE != K21_MHA) s *= MODE == K21_DOT ? mul : wc;
      if (a.masked && !mha_keep(a, row.b, t0 + j, row.w)) s += MHA_MASK_ADDER;
      const float p = __fdividef(expf(s - sM[(base + j) * 2]), sM[(base + j) * 2 + 1]);
      float dp = team_dot<E>(v, gr, dv, lane), pz = p;
      if (drop) {
        const float z = zr[j] ? a.drop_scale : 0.f;
        pz = p * z;
        dp *= z;
      }
      const float ds = p * (dp - sD[base + j]);
      const float f = ds * wc * c;                   // K25: dS/dk_d = wc c w_d (1 - t_d^2)
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dv) gv[i] = fmaf(pz, gr[d], gv[i]);
        if constexpr (MODE == K25_TANH) gk[i] = fmaf(f * w[i], fmaf(-t[i], t[i], 1.f), gk[i]);
        else if (d < dk) gk[i] = fmaf(ds, qr[d], gk[i]);
      }
    }
  }
  if (!row.live) return;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if (d < dk) a.dk_out[kb + d] = MODE == K21_DOT ? gk[i] * mul : gk[i];
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

// The dense modes' dQ: as mha_bwd_q_kernel, with z dO.v - delta taken as dO.(z v - O), and the per-row partials of the
// score weights' gradients when a.part is set: dot [rows] = sum_j ds_j q . k_j; concat [2][rows] =
// (sum_j ds_j wc sum_d (q_d + k_d)(1 - t_d^2), sum_j ds_j sum_d t_d); additive [rows][dk] = sum_j ds_j t_d
template <int E, int MODE>
__global__ void __launch_bounds__(MHA_THREADS, 1)
dense_bwd_q_kernel(const MhaArgs a) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x % MHA_LANES, T = a.T, S = a.S, H = a.H, dk = a.dk, dv = a.dv;
  const int rows = (int)(a.B * H * T);
  const MhaRow row(rows, T, H);
  const int n0 = blockIdx.x * MHA_TEAMS / T;
  float* sK = sm;
  float* sV = sm + (size_t)a.nseq * a.tile * dk;
  uint8_t* sZ = reinterpret_cast<uint8_t*>(sV + (size_t)a.nseq * a.tile * dv);
  const uint8_t* zr = sZ + (threadIdx.x / MHA_LANES) * a.tile;
  const bool drop = a.drop;

  float q[E], g[E], o[E], gq[E], w[E], t[E], pa[E], mul, c, wc;
  dense_weights<E, MODE>(a, lane, mul, w, c, wc);
  const long long qb = (((long long)row.b * T + row.w) * H + row.h) * (long long)dk;
  const long long ob = (((long long)row.b * T + row.w) * H + row.h) * (long long)dv;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    q[i] = d < dk ? a.q[qb + d] : 0.f;
    g[i] = d < dv ? a.dout[ob + d] : 0.f;
    o[i] = d < dv ? a.o[ob + d] : 0.f;
    gq[i] = pa[i] = 0.f;
  }
  float mx = a.stats[2ll * row.r];
  const float l = a.stats[2ll * row.r + 1];
  // The weight gradients' partials sum ds_j (raw_j - cr): sum_j ds_j = 0, so any constant cr leaves them unchanged, and
  // cr = the row max in raw units keeps raw_j - cr small where ds_j is large
  const float post = MODE == K21_DOT ? mul : wc, mu = mx < 0.5f * MHA_MASK_ADDER ? mx - MHA_MASK_ADDER : mx;
  const float cr = post != 0.f ? mu / post : 0.f;
  if (!dense_out_kept(a, row.r)) mx = INFINITY;      // an output-masked query row: p = 0, no gradient
  float pc = 0.f, pw = 0.f;
  for (int s0 = 0; s0 < S; s0 += a.tile) {
    const int sn = min(a.tile, S - s0);
    __syncthreads();
    mha_stage(sK, a.k, n0, row.nseq, s0, sn, S, H, dk, a.tile, 1.f);
    mha_stage(sV, a.v, n0, row.nseq, s0, sn, S, H, dv, a.tile, 1.f);
    if (drop) dense_keep_query_rows(sZ, a, rows, s0, sn);
    __syncthreads();
    const float* kr = sK + (size_t)row.slot * a.tile * dk;
    const float* vr = sV + (size_t)row.slot * a.tile * dv;
    for (int j = 0; j < sn; ++j) {
      const float raw = mha_score<E, MODE>(q, kr + j * dk, dk, lane, w, c, t);
      float s = raw * post;
      if (a.masked && !mha_keep(a, row.b, row.w, s0 + j)) s += MHA_MASK_ADDER;
      const float p = __fdividef(expf(s - mx), l);
      // z dO.v_j - delta = dO.(z v_j - O): no cancellation between two rounded dot products
      const float z = drop ? (zr[j] ? a.drop_scale : 0.f) : 1.f;
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const int d = lane + MHA_LANES * i;
        if (d < dv) acc = fmaf(g[i], fmaf(z, vr[j * dv + d], -o[i]), acc);
      }
      const float ds = p * team_sum(acc);
      if constexpr (MODE == K25_TANH) {
        const float f = ds * wc * c;
        float u = 0.f;
#pragma unroll
        for (int i = 0; i < E; ++i) {
          const int d = lane + MHA_LANES * i;
          const float dt = fmaf(-t[i], t[i], 1.f);
          gq[i] = fmaf(f * w[i], dt, gq[i]);
          pa[i] = fmaf(ds, t[i], pa[i]);
          if (d < dk) u = fmaf(q[i] + kr[j * dk + d], dt, u);
        }
        pc = fmaf(ds * wc, u, pc);
        pw = fmaf(ds, raw - cr, pw);
      } else {
#pragma unroll
        for (int i = 0; i < E; ++i) {
          const int d = lane + MHA_LANES * i;
          if (d < dk) gq[i] = fmaf(ds, kr[j * dk + d], gq[i]);
        }
        pw = fmaf(ds, raw - cr, pw);
      }
    }
  }
  if constexpr (MODE == K21_DOT) {
    if (a.part && row.live && lane == 0) a.part[row.r] = pw;   // d scale = sum_j ds_j q . k_j
  } else if constexpr (MODE == K25_TANH) {
    if (a.part) {
      if (a.additive) {
#pragma unroll
        for (int i = 0; i < E; ++i) {
          const int d = lane + MHA_LANES * i;
          if (row.live && d < dk) a.part[(long long)row.r * dk + d] = pa[i];
        }
      } else {
        pc = team_sum(pc);
        if (row.live && lane == 0) {
          a.part[row.r] = pc;
          a.part[rows + row.r] = pw;
        }
      }
    }
  }
  if (!row.live) return;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    const int d = lane + MHA_LANES * i;
    if (d < dk) a.dq[qb + d] = MODE == K25_TANH ? gq[i] : gq[i] * mul;
  }
}

// The staged-tile plan: how many sequences 32 consecutive rows of length L can touch, and how many rows per sequence
// fit the shared-memory budget at `width` floats per staged row.
static inline void mha_plan(int L, int width, int* nseq, int* tile, size_t* smem) {
  const long long span = (MHA_TEAMS - 1 + L - 1) / L + 1;
  *nseq = (int)(span < MHA_TEAMS ? span : MHA_TEAMS);
  long long t = MHA_SMEM_BUDGET / ((long long)*nseq * width * 4);
  t = t < 1 ? 1 : (t > MHA_MAX_TILE ? MHA_MAX_TILE : t);
  *tile = (int)t;
  *smem = (size_t)*nseq * *tile * width * 4;
}

// head elements per lane: E * 8 >= max(dk, dv), E a power of two naming one kernel instance
static inline int mha_elems(int dk, int dv) {
  const int w = dk > dv ? dk : dv;
  int e = 1;
  while (e * MHA_LANES < w) e *= 2;
  return e;
}

enum { MHA_FWD, MHA_BWD_KV, MHA_BWD_Q };

// The opt-in shared-memory cap is set once per device and call site, so it is the plan's budget (plus the dense modes'
// keep bytes), which every plan fits
template <int E, int MODE>
static int mha_launch_e(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  constexpr int cap = MHA_SMEM_BUDGET + (MODE == K21_MHA ? 0 : MHA_KEEP_BYTES);
  switch (which) {
    case MHA_FWD:
      TFRS_DYN_SMEM((mha_fwd_kernel<E, MODE>), cap);
      mha_fwd_kernel<E, MODE><<<grid, MHA_THREADS, smem, st>>>(a);
      break;
    case MHA_BWD_KV:
      TFRS_DYN_SMEM((mha_bwd_kv_kernel<E, MODE>), cap);
      mha_bwd_kv_kernel<E, MODE><<<grid, MHA_THREADS, smem, st>>>(a);
      break;
    default:
      if constexpr (MODE == K21_MHA) {
        TFRS_DYN_SMEM(mha_bwd_q_kernel<E>, cap);
        mha_bwd_q_kernel<E><<<grid, MHA_THREADS, smem, st>>>(a);
      } else {
        TFRS_DYN_SMEM((dense_bwd_q_kernel<E, MODE>), cap);
        dense_bwd_q_kernel<E, MODE><<<grid, MHA_THREADS, smem, st>>>(a);
      }
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

template <int MODE>
static int mha_launch_mode(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  switch (mha_elems(a.dk, a.dv)) {
    case 1: return mha_launch_e<1, MODE>(which, a, grid, smem, st);
    case 2: return mha_launch_e<2, MODE>(which, a, grid, smem, st);
    case 4: return mha_launch_e<4, MODE>(which, a, grid, smem, st);
    case 8: return mha_launch_e<8, MODE>(which, a, grid, smem, st);
    case 16: return mha_launch_e<16, MODE>(which, a, grid, smem, st);
  }
  set_error("attention: no kernel instance for dk = %d, dv = %d", a.dk, a.dv);
  return TFRS_ERR_INVALID_ARG;
}

// K25's instances (additive_attention.cu)
int k25_launch(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st);

}  // namespace tfrs
