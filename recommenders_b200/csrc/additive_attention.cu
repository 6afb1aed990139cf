// additive_attention.cu -- K25: the tanh scores of tf.keras.layers.Attention(score_mode="concat") and
// AdditiveAttention, s = wc * sum_d w_d tanhf(c (q_d + k_d)) with (w = 1, c = scale, wc = concat_score_weight) for concat
// and (w = scale, c = 1, wc = 1) for additive, on K21's team-per-row kernels (attention.cuh): the same staged tiles,
// online softmax, mask and dropout rules.  tanhf, not tanh.approx: its ~2^-11 relative error would show in the scores.
// Each lane keeps the tanh of its elements of the current score in registers, so the backward's dS/dq_d = dS/dk_d =
// wc c w_d (1 - t_d^2) reuses them and no [B, Tq, Tv, d] tensor is ever written; dq and dk accumulate in registers.
// The entry points are attention.cu's tfrs_dense_attention_*.
#include "attention.cuh"

namespace tfrs {

int k25_launch(int which, const MhaArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
  return mha_launch_mode<K25_TANH>(which, a, grid, smem, st);
}

}  // namespace tfrs
