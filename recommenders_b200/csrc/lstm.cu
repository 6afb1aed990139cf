// lstm.cu -- K20: the recurrence of tf.keras.layers.LSTM (TF2 defaults: tanh / sigmoid, one bias), the cell users put in
// the sequential retrieval tutorial's query tower instead of the GRU: LstmCell on rnn.cuh's kernels.  gx = x.W + b; the
// chains give z = h_{t-1}.U for the columns (i, f, c, o).
//   forward: the cell state c lives in registers; saves (i, f, g, o), c_t and h_{t-1} per step.
//   backward: dh and dc in registers; the gate gradients dz go to HBM (they are both the projection's and U's output
//     gradient) and to shared memory, then dh <- dz.U^T and dc <- dc f.  The same C entry then runs K6's backward for
//     dU = h_{t-1}^T . dz.
#include "rnn.cuh"

namespace tfrs {

struct LstmCell {
  static constexpr int NG = 4;
  using State = float;   // c in the forward, dc in the backward

  struct FwdArgs : RnnFwdArgs {
    const float* c0; float* c_last; float* gates; float* c_seq; float* h_prev;
  };

  struct BwdArgs : RnnBwdArgs {
    const float* gates; const float* c_seq; const float* c0; const float* g_h; const float* g_c;
    float* dz; float* dc0;
  };

  static __device__ __forceinline__ void fwd_init(const FwdArgs& p, float& c, long long b, int j) {
    c = (p.c0 && b < p.B && j < p.u) ? p.c0[b * p.u + j] : 0.f;
  }

  static __device__ __forceinline__ float fwd_gates(const FwdArgs& p, float& c, const float (&acc)[NG], long long o, int j,
                                                    float) {
    const int u = p.u, u4 = 4 * u;
    const float* z = p.gx + o * u4;
    const float ig = rnn_sigmoid(z[j] + acc[0]);
    const float fg = rnn_sigmoid(z[u + j] + acc[1]);
    const float gg = rnn_tanh(z[2 * u + j] + acc[2]);
    const float og = rnn_sigmoid(z[3 * u + j] + acc[3]);
    c = fg * c + ig * gg;
    const float h = og * rnn_tanh(c);
    if (p.gates) {
      float* gt = p.gates + o * u4;
      gt[j] = ig; gt[u + j] = fg; gt[2 * u + j] = gg; gt[3 * u + j] = og;
    }
    return h;
  }

  static __device__ __forceinline__ void fwd_save(const FwdArgs& p, float c, long long o, int j, float hp) {
    if (p.gates) {
      p.c_seq[o * p.u + j] = c;
      p.h_prev[o * p.u + j] = hp;
    }
  }

  static __device__ __forceinline__ void fwd_last(const FwdArgs& p, float c, long long bj) { p.c_last[bj] = c; }

  static __device__ __forceinline__ float bwd_gates(const BwdArgs& p, float& dc, float d, bool keep, long long b,
                                                    long long o, int j, long long t, float* sgr) {
    const int u = p.u, u4 = 4 * u;
    if (t == p.T - 1) {
      if (p.g_h) d += p.g_h[b * u + j];
      if (p.g_c) dc += p.g_c[b * u + j];
    }
    float di = 0.f, df = 0.f, dgg = 0.f, dout = 0.f;
    if (keep) {
      const float* gt = p.gates + o * u4;
      const float ig = gt[j], fg = gt[u + j], gg = gt[2 * u + j], og = gt[3 * u + j];
      const float cp = t > 0 ? p.c_seq[(o - 1) * u + j] : (p.c0 ? p.c0[b * u + j] : 0.f);
      const float tc = rnn_tanh(p.c_seq[o * u + j]);
      dout = d * tc * rnn_sigmoid_grad(og);
      const float dct = dc + d * og * rnn_tanh_grad(tc);
      di = dct * gg * rnn_sigmoid_grad(ig);
      df = dct * cp * rnn_sigmoid_grad(fg);
      dgg = dct * ig * rnn_tanh_grad(gg);
      dc = dct * fg;
    }
    float* dzr = p.dz + o * u4;
    dzr[j] = di; dzr[u + j] = df; dzr[2 * u + j] = dgg; dzr[3 * u + j] = dout;
    sgr[j] = di; sgr[u + j] = df; sgr[2 * u + j] = dgg; sgr[3 * u + j] = dout;
    return d;
  }

  // acc alone, not carry + acc: a kept step's dh_{t-1} is dz.U^T only, and +0 + acc would turn an acc of -0 into +0
  static __device__ __forceinline__ void bwd_dh(bool keep, float& dh, float acc) {
    if (keep) dh = acc;
  }

  static __device__ __forceinline__ bool bwd_initial(const BwdArgs& p) { return p.dh0 || p.dc0; }

  static __device__ __forceinline__ void bwd_last(const BwdArgs& p, float dc, long long bj) {
    if (p.dc0) p.dc0[bj] = dc;
  }
};

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_lstm_fwd_f32(const float* gx, const float* U, const float* h0, const float* c0, const void* mask,
                                 int mask_kind, int64_t B, int64_t T, int units, float* out_seq, float* h_last,
                                 float* c_last, float* gates, float* c_seq, float* h_prev, void* stream) {
  int rc = rnn_check("lstm_fwd", B, T, units, TFRS_LSTM_MAX_UNITS, mask, mask_kind);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(gx && U && h_last && c_last, "lstm_fwd: NULL pointer");
  TFRS_CHECK_ARG(!gates == !c_seq && !gates == !h_prev, "lstm_fwd: gates, c_seq and h_prev are saved together");
  const RnnTile tl = rnn_tile(units);
  LstmCell::FwdArgs a{{gx, U, h0, mask, B, T, units, tl.jt, 0, out_seq, h_last}, c0, c_last, gates, c_seq, h_prev};
  size_t smem;
  rnn_smem(2 * tl.rows * units, units, 4 * units, &a.ks, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  return rnn_dispatch<LstmCell>("lstm_fwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
}

extern "C" size_t tfrs_lstm_bwd_workspace_bytes(int64_t B, int64_t T, int units) {
  if (B <= 0 || T <= 0 || units <= 0) return 256;
  const size_t k6 = tfrs_dense_bwd_workspace_bytes((long long)B * T, units, 4 * units);
  return k6 < 256 ? 256 : k6;
}

extern "C" int tfrs_lstm_bwd_f32(const float* U, const float* gates, const float* c_seq, const float* h_prev,
                                 const float* c0, const void* mask, int mask_kind, const float* g_seq, const float* g_h,
                                 const float* g_c, int64_t B, int64_t T, int units, float* dz, float* dU, float* dh0,
                                 float* dc0, void* ws, size_t ws_bytes, void* stream) {
  int rc = rnn_check("lstm_bwd", B, T, units, TFRS_LSTM_MAX_UNITS, mask, mask_kind);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(U && gates && c_seq && dz, "lstm_bwd: NULL pointer");
  TFRS_CHECK_ARG(!dU || h_prev, "lstm_bwd: dU needs h_prev");
  const size_t need = tfrs_lstm_bwd_workspace_bytes(B, T, units);
  if (dU && (!ws || ws_bytes < need)) { set_error("lstm_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "lstm_bwd: workspace must be 16-byte aligned");
  const RnnTile tl = rnn_tile(units);
  LstmCell::BwdArgs a{{U, mask, g_seq, B, T, units, tl.jt, 0, dh0}, gates, c_seq, c0, g_h, g_c, dz, dc0};
  size_t smem;
  rnn_smem(2 * tl.rows * 4 * units, 4 * units, units + 1, &a.cs, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  rc = rnn_dispatch<LstmCell>("lstm_bwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
  if (rc || !dU) return rc;
  // dU = h_prev^T . dz: K6's backward of a linear layer whose output gradient is dz
  return tfrs_dense_bwd_f32(h_prev, U, dz, dz, nullptr, (long long)B * T, units, 4 * units, TFRS_ACT_LINEAR, nullptr, dU,
                            nullptr, ws, ws_bytes, stream);
}
