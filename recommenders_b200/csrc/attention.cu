// attention.cu -- K21: the attention core of tf.keras.layers.MultiHeadAttention (attention_axes over the sequence, no
// dropout), and the dot-score mode of the dense attention layers (tf.keras.layers.Attention), whose entry points also
// dispatch K25's tanh scores (additive_attention.cu).  The kernels are attention.cuh's.  The Q / K / V / output
// projections of MultiHeadAttention are K6 (dense.cu) and run around this file; here Q [B, T, H*dk], K [B, S, H*dk]
// and V [B, S, H*dv] are read in place (head h is columns h*dk .. h*dk + dk - 1 of a row), with no head transpose.
#include "attention.cuh"

namespace tfrs {

static int mha_check(const char* what, int64_t B, int64_t T, int64_t S, int H, int dk, int dv, const TfrsMhaMasks* m) {
  TFRS_CHECK_ARG(B >= 0 && T >= 1 && S >= 1 && H >= 1 && B < (1ll << 31) && T < (1ll << 31) && S < (1ll << 31) &&
                     B * H * (T > S ? T : S) < (1ll << 31),
                 "%s: bad shape B=%lld T=%lld S=%lld H=%d", what, (long long)B, (long long)T, (long long)S, H);
  TFRS_CHECK_ARG(dk >= 1 && dk <= TFRS_MHA_MAX_HEAD_DIM && dv >= 1 && dv <= TFRS_MHA_MAX_HEAD_DIM,
                 "%s: key_dim = %d and value_dim = %d must be in 1 .. %d", what, dk, dv, TFRS_MHA_MAX_HEAD_DIM);
  if (m) {
    const void* ps[4] = {m->query, m->value, m->key, m->attention};
    const int ks[4] = {m->query_kind, m->value_kind, m->key_kind, m->attention_kind};
    for (int i = 0; i < 4; ++i) TFRS_CHECK_MASK(what, ps[i], ks[i]);
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

static int dense_check(const char* what, int64_t B, int64_t Tq, int64_t Tv, int dim, int dv,
                       const TfrsDenseAttention* d) {
  TFRS_CHECK_ARG(d, "%s: NULL descriptor", what);
  TFRS_CHECK_ARG(d->mode == TFRS_DENSE_DOT || d->mode == TFRS_DENSE_CONCAT || d->mode == TFRS_DENSE_ADDITIVE,
                 "%s: unknown score mode %d", what, d->mode);
  TFRS_CHECK_ARG(d->mode != TFRS_DENSE_CONCAT || d->concat_weight, "%s: concat scores need concat_weight", what);
  TFRS_CHECK_ARG(d->rate >= 0.0 && d->rate < 1.0, "%s: dropout must be in [0, 1), got %g", what, d->rate);
  TfrsMhaMasks m{};
  m.query = d->query_mask; m.query_kind = d->query_mask_kind;
  m.value = d->value_mask; m.value_kind = d->value_mask_kind;
  return mha_check(what, B, Tq, Tv, 1, dim, dv, &m);
}

// one head over the B * Tq query rows; the query mask leaves the softmax and masks the output rows instead
static MhaArgs dense_args(const float* Q, const float* K, const float* V, const TfrsDenseAttention* d, int64_t B,
                          int64_t Tq, int64_t Tv, int dim, int dv) {
  MhaArgs a{};
  a.q = Q; a.k = K; a.v = V;
  a.m.value = d->value_mask; a.m.value_kind = d->value_mask_kind;
  a.m.causal = d->causal;
  a.masked = a.m.value || a.m.causal;
  a.B = B; a.T = (int)Tq; a.S = (int)Tv; a.H = 1; a.dk = dim; a.dv = dv;
  a.scale = 1.f;
  a.score_scale = d->scale;
  a.concat_weight = d->mode == TFRS_DENSE_CONCAT ? d->concat_weight : nullptr;
  a.additive = d->mode == TFRS_DENSE_ADDITIVE;
  a.omask = d->query_mask; a.omask_kind = d->query_mask_kind;
  a.drop = d->rate > 0.0;
  if (a.drop) {
    a.thr = (uint32_t)ceil(d->rate * 16777216.0);
    a.drop_scale = (float)(1.0 / (1.0 - d->rate));
    a.k0 = (uint32_t)d->seed; a.k1 = (uint32_t)(d->seed >> 32);
    a.c0 = (uint32_t)d->call; a.c1 = (uint32_t)(d->call >> 32);
  }
  return a;
}

static int dense_launch(int mode, int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  smem += (size_t)MHA_TEAMS * a.tile;                // the keep bytes
  return mode == TFRS_DENSE_DOT ? mha_launch_mode<K21_DOT>(which, a, grid, smem, st)
                                : k25_launch(which, a, grid, smem, st);
}

// the per-row partials of the score weights' gradients: one column (dot), two (concat) or dim (additive)
static long long dense_part_cols(int mode, int dim) {
  return mode == TFRS_DENSE_DOT ? 1 : mode == TFRS_DENSE_CONCAT ? 2 : dim;
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
  return mha_launch_mode<K21_MHA>(MHA_FWD, a, (unsigned)ceil_div(B * H * T, MHA_TEAMS), smem, (cudaStream_t)stream);
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
  if ((rc = mha_launch_mode<K21_MHA>(MHA_BWD_KV, a, kgrid, smem, st))) return rc;
  mha_plan((int)T, dk + dv, &a.nseq, &a.tile, &smem);
  return mha_launch_mode<K21_MHA>(MHA_BWD_Q, a, qgrid, smem, st);
}

extern "C" int tfrs_dense_attention_fwd_f32(const float* Q, const float* K, const float* V,
                                            const TfrsDenseAttention* desc, int64_t B, int64_t Tq, int64_t Tv, int dim,
                                            int dv, float* O, float* stats, float* P, void* stream) {
  int rc = dense_check("dense_attention_fwd", B, Tq, Tv, dim, dv, desc);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(Q && K && V && O, "dense_attention_fwd: NULL pointer");
  MhaArgs a = dense_args(Q, K, V, desc, B, Tq, Tv, dim, dv);
  a.out = O; a.stats_out = stats; a.p = P;
  size_t smem;
  mha_plan((int)Tq, dim + dv, &a.nseq, &a.tile, &smem);
  return dense_launch(desc->mode, MHA_FWD, a, (unsigned)ceil_div(B * Tq, MHA_TEAMS), smem, (cudaStream_t)stream);
}

extern "C" size_t tfrs_dense_attention_bwd_workspace_bytes(int mode, int64_t B, int64_t Tq, int dim) {
  const long long n = B > 0 && Tq > 0 ? B * Tq : 0;
  const size_t bytes = align_up((size_t)n * 4, 256) + align_up((size_t)(n * dense_part_cols(mode, dim > 0 ? dim : 0)) * 4, 256);
  return bytes < 256 ? 256 : bytes;
}

extern "C" int tfrs_dense_attention_bwd_f32(const float* Q, const float* K, const float* V,
                                            const TfrsDenseAttention* desc, const float* O, const float* stats,
                                            const float* dO, int64_t B, int64_t Tq, int64_t Tv, int dim, int dv,
                                            float* dQ, float* dK, float* dV, float* dscale, float* dconcat_weight,
                                            void* ws, size_t ws_bytes, void* stream) {
  int rc = dense_check("dense_attention_bwd", B, Tq, Tv, dim, dv, desc);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(Q && K && V && O && stats && dO && dQ && dK && dV, "dense_attention_bwd: NULL pointer");
  TFRS_CHECK_ARG(!dconcat_weight || desc->mode == TFRS_DENSE_CONCAT,
                 "dense_attention_bwd: dconcat_weight is for concat scores");
  if (!ws || ws_bytes < tfrs_dense_attention_bwd_workspace_bytes(desc->mode, B, Tq, dim)) {
    set_error("dense_attention_bwd: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "dense_attention_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = B * Tq;
  MhaArgs a = dense_args(Q, K, V, desc, B, Tq, Tv, dim, dv);
  a.o = O; a.dout = dO; a.stats = stats; a.delta = static_cast<float*>(ws); a.delta_out = static_cast<float*>(ws);
  a.dq = dQ; a.dk_out = dK; a.dv_out = dV;
  float* part = reinterpret_cast<float*>(static_cast<char*>(ws) + align_up((size_t)rows * 4, 256));
  a.part = dscale || dconcat_weight ? part : nullptr;
  const unsigned qgrid = (unsigned)ceil_div(rows, MHA_TEAMS), kgrid = (unsigned)ceil_div(B * Tv, MHA_TEAMS);
  mha_delta_kernel<<<qgrid, MHA_THREADS, 0, st>>>(a);
  TFRS_LAUNCH_CHECK();
  size_t smem;
  mha_plan((int)Tv, dim + dv + 3, &a.nseq, &a.tile, &smem);
  if ((rc = dense_launch(desc->mode, MHA_BWD_KV, a, kgrid, smem, st))) return rc;
  mha_plan((int)Tq, dim + dv, &a.nseq, &a.tile, &smem);
  if ((rc = dense_launch(desc->mode, MHA_BWD_Q, a, qgrid, smem, st))) return rc;
  // the fixed-order folds of the per-row partials
  if (desc->mode == TFRS_DENSE_ADDITIVE) {
    if (dscale && (rc = reduce_columns(part, rows, dim, dscale, st))) return rc;
  } else {
    if (dscale && (rc = reduce_loss(part, rows, 1, dscale, st))) return rc;
    if (dconcat_weight && (rc = reduce_loss(part + rows, rows, 1, dconcat_weight, st))) return rc;
  }
  return TFRS_OK;
}
