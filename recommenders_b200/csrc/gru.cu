// gru.cu -- K19: the recurrence of tf.keras.layers.GRU (reset_after=True, the TF2 default) as the reference's sequential
// retrieval tutorial builds its query tower (`Sequential([StringLookup, Embedding, GRU(32)])`): GruCell on rnn.cuh's
// kernels.  gx = x.W + b_i; the chains give gr = h_{t-1}.U (+ b_r) for the columns (z, r, h).
//   forward: saves (z, r, hh, gr_h) and h_{t-1} per step; no state beyond h.
//   backward: dh <- dh z + dgr.U^T, dgr = (dz, dr, dgh) staged in shared memory; the gradient of gx, (dz, dr, dhp), and
//     dgr go to HBM.  The same C entry then runs K6's backward for dU = h_{t-1}^T . dgr and db_r = colsum(dgr).
#include "rnn.cuh"

namespace tfrs {

struct GruCell {
  static constexpr int NG = 3;
  struct State {};

  struct FwdArgs : RnnFwdArgs {
    const float* br; float* gates; float* h_prev;
  };

  struct BwdArgs : RnnBwdArgs {
    const float* gates; const float* h_prev; const float* g_last;
    float* dgx; float* dgr;
  };

  static __device__ __forceinline__ void fwd_init(const FwdArgs&, State&, long long, int) {}

  static __device__ __forceinline__ float fwd_gates(const FwdArgs& p, State&, const float (&acc)[NG], long long o, int j,
                                                    float hp) {
    const int u = p.u, u3 = 3 * u;
    const float* gxr = p.gx + o * u3;
    float gz = acc[0], gr = acc[1], gh = acc[2];
    if (p.br) { gz += __ldg(p.br + j); gr += __ldg(p.br + u + j); gh += __ldg(p.br + 2 * u + j); }
    const float z = rnn_sigmoid(gxr[j] + gz);
    const float r = rnn_sigmoid(gxr[u + j] + gr);
    const float hh = rnn_tanh(gxr[2 * u + j] + r * gh);
    const float h = z * hp + (1.f - z) * hh;
    if (p.gates) {
      float* gt = p.gates + o * 4 * u;
      gt[j] = z; gt[u + j] = r; gt[2 * u + j] = hh; gt[3 * u + j] = gh;
    }
    return h;
  }

  static __device__ __forceinline__ void fwd_save(const FwdArgs& p, const State&, long long o, int j, float hp) {
    if (p.h_prev) p.h_prev[o * p.u + j] = hp;
  }

  static __device__ __forceinline__ void fwd_last(const FwdArgs&, const State&, long long) {}

  static __device__ __forceinline__ float bwd_gates(const BwdArgs& p, State&, float d, bool keep, long long b,
                                                    long long o, int j, long long t, float* sgr) {
    const int u = p.u, u3 = 3 * u;
    if (p.g_last && t == p.T - 1) d += p.g_last[b * u + j];
    float dz = 0.f, dr = 0.f, dhp = 0.f, dgh = 0.f, carry = d;
    if (keep) {
      const float* gt = p.gates + o * 4 * u;
      const float z = gt[j], r = gt[u + j], hh = gt[2 * u + j], grh = gt[3 * u + j];
      const float hp = p.h_prev[o * u + j];
      dz = d * (hp - hh) * rnn_sigmoid_grad(z);
      dhp = d * (1.f - z) * rnn_tanh_grad(hh);
      dr = dhp * grh * rnn_sigmoid_grad(r);
      dgh = dhp * r;
      carry = d * z;
    }
    float* gx = p.dgx + o * u3;
    float* gr = p.dgr + o * u3;
    gx[j] = dz; gx[u + j] = dr; gx[2 * u + j] = dhp;
    gr[j] = dz; gr[u + j] = dr; gr[2 * u + j] = dgh;
    const float dg[NG] = {dz, dr, dgh};   // stored through a loop: three direct stores compile to other code
#pragma unroll
    for (int q = 0; q < NG; ++q) sgr[q * u + j] = dg[q];
    return carry;
  }

  // carry + acc, not acc alone: the d z of a kept step is part of dh_{t-1}
  static __device__ __forceinline__ void bwd_dh(bool keep, float& dh, float acc) { dh = keep ? dh + acc : dh; }

  static __device__ __forceinline__ bool bwd_initial(const BwdArgs& p) { return p.dh0 != nullptr; }

  static __device__ __forceinline__ void bwd_last(const BwdArgs&, const State&, long long) {}
};

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_gru_fwd_f32(const float* gx, const float* U, const float* b_r, const float* h0, const void* mask,
                                int mask_kind, int64_t B, int64_t T, int units, float* out_seq, float* h_last, float* gates,
                                float* h_prev, void* stream) {
  int rc = rnn_check("gru_fwd", B, T, units, TFRS_GRU_MAX_UNITS, mask, mask_kind);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(gx && U && h_last, "gru_fwd: NULL pointer");
  TFRS_CHECK_ARG(!gates == !h_prev, "gru_fwd: gates and h_prev are saved together");
  const RnnTile tl = rnn_tile(units);
  GruCell::FwdArgs a{{gx, U, h0, mask, B, T, units, tl.jt, 0, out_seq, h_last}, b_r, gates, h_prev};
  size_t smem;
  rnn_smem(2 * tl.rows * units, units, 3 * units, &a.ks, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  return rnn_dispatch<GruCell>("gru_fwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
}

extern "C" size_t tfrs_gru_bwd_workspace_bytes(int64_t B, int64_t T, int units) {
  if (B <= 0 || T <= 0 || units <= 0) return 256;
  const long long n = (long long)B * T;
  return align_up((size_t)n * 3 * units * 4, 1024) + tfrs_dense_bwd_workspace_bytes(n, units, 3 * units);
}

extern "C" int tfrs_gru_bwd_f32(const float* U, const float* gates, const float* h_prev, const void* mask, int mask_kind,
                                const float* g_seq, const float* g_last, int64_t B, int64_t T, int units, float* dgx,
                                float* dU, float* db_r, float* dh0, void* ws, size_t ws_bytes, void* stream) {
  int rc = rnn_check("gru_bwd", B, T, units, TFRS_GRU_MAX_UNITS, mask, mask_kind);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  TFRS_CHECK_ARG(U && gates && h_prev && dgx, "gru_bwd: NULL pointer");
  const size_t need = tfrs_gru_bwd_workspace_bytes(B, T, units);
  if (!ws || ws_bytes < need) { set_error("gru_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "gru_bwd: workspace must be 16-byte aligned");
  const long long n = (long long)B * T;
  float* dgr = (float*)ws;
  unsigned char* kws = (unsigned char*)ws + align_up((size_t)n * 3 * units * 4, 1024);
  const RnnTile tl = rnn_tile(units);
  GruCell::BwdArgs a{{U, mask, g_seq, B, T, units, tl.jt, 0, dh0}, gates, h_prev, g_last, dgx, dgr};
  size_t smem;
  rnn_smem(2 * tl.rows * 3 * units, 3 * units, units + 1, &a.cs, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  rc = rnn_dispatch<GruCell>("gru_bwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
  if (rc || (!dU && !db_r)) return rc;
  // dU = h_prev^T . dgr, db_r = colsum(dgr): K6's backward of a linear layer whose output gradient is dgr
  return tfrs_dense_bwd_f32(h_prev, U, dgr, dgr, nullptr, n, units, 3 * units, TFRS_ACT_LINEAR, nullptr, dU, db_r, kws,
                            ws_bytes - (size_t)(kws - (unsigned char*)ws), stream);
}
