// lstm.cu -- K20: the recurrence of tf.keras.layers.LSTM (TF2 defaults: tanh / sigmoid, one bias), the cell users put in
// the sequential retrieval tutorial's query tower instead of the GRU.  The input projection gx = x.W + b is K6
// (dense.cu) and comes in precomputed; this file owns the T-step recurrence, one launch each way.  The row-tile plan,
// mask test, shared-memory budget and instance dispatch are K19's (rnn.cuh).
//
//   Each CTA owns a tile of R batch rows for the whole sequence; rows are independent, so the only synchronisation is
//   __syncthreads.  Thread (j0, g) owns hidden units j = j0 + JT*a (a < UJ) of the tile rows g + G*i (i < RJ) at every
//   step, so h is double-buffered in shared memory (R * u <= 2048: at most 16 KB) and c never leaves registers.
//   forward, per step: z = h_{t-1}.U as four fmaf chains (columns i, f, c, o) over k ascending from +0.0f, the h tile
//     and U read from shared memory (U resident when its 16 u^2 bytes fit, otherwise streamed from L2 in k-slices every
//     step); then the gate epilogue adds gx, updates c in registers and writes h_t into the other h buffer.
//   backward, per step in reverse: dh and dc in registers; the gate gradients dz of every owned pair go to HBM (they
//     are both the projection's and U's output gradient) and to shared memory (two buffers, so one barrier per step),
//     then dh <- dz.U^T as the fmaf chain over the 4u columns ascending, U^T staged transposed, and dc <- dc f.  The
//     same C entry then runs K6's backward for dU = h_{t-1}^T . dz.
//   A masked step does no arithmetic: the forward carries h and c, the backward passes dh and dc through and writes
//   zero rows.
#include "rnn.cuh"

namespace tfrs {

struct LstmFwdArgs {
  const float* gx; const float* U; const float* h0; const float* c0; const void* mask;
  long long B, T; int u, jt, ks;
  float* seq; float* h_last; float* c_last; float* gates; float* c_seq; float* h_prev;
};

struct LstmBwdArgs {
  const float* U; const float* gates; const float* c_seq; const float* c0; const void* mask;
  const float* g_seq; const float* g_h; const float* g_c;
  long long B, T; int u, jt, cs;
  float* dz; float* dh0; float* dc0;
};

template <typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
lstm_fwd_kernel(const LstmFwdArgs p) {
  extern __shared__ float sm[];
  const int u = p.u, u4 = 4 * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
  const int j0 = threadIdx.x % JT, g = threadIdx.x / JT;
  const long long b0 = (long long)blockIdx.x * R;
  float* sU = sm + 2 * R * u;
  const bool resident = p.ks >= u;

  for (int e = threadIdx.x; e < R * u; e += RNN_THREADS) {
    const long long b = b0 + e / u;
    sm[e] = (p.h0 && b < p.B) ? p.h0[b * u + e % u] : 0.f;
    sm[R * u + e] = 0.f;
  }
  if (resident)
    for (int e = threadIdx.x; e < u * u4; e += RNN_THREADS) sU[e] = __ldg(p.U + e);
  float c[UJ][RJ];
#pragma unroll
  for (int i = 0; i < RJ; ++i) {
    const long long b = b0 + g + G * i;
#pragma unroll
    for (int a = 0; a < UJ; ++a) {
      const int j = j0 + JT * a;
      c[a][i] = (p.c0 && b < p.B && j < u) ? p.c0[b * u + j] : 0.f;
    }
  }
  __syncthreads();

  int cur = 0;
  for (long long t = 0; t < p.T; ++t) {
    const float* hc = sm + cur * R * u;
    float* hn = sm + (cur ^ 1) * R * u;
    float acc[UJ][RJ][4];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) acc[a][i][0] = acc[a][i][1] = acc[a][i][2] = acc[a][i][3] = 0.f;

    for (int k0 = 0; k0 < u; k0 += p.ks) {
      const int kn = min(p.ks, u - k0);
      if (!resident) {
        __syncthreads();
        const float* src = p.U + (long long)k0 * u4;
        for (int e = threadIdx.x; e < kn * u4; e += RNN_THREADS) sU[e] = __ldg(src + e);
        __syncthreads();
      }
      const float* w = resident ? sU + (long long)k0 * u4 : sU;
      for (int kk = 0; kk < kn; ++kk) {
        float hv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) hv[i] = hc[(g + G * i) * u + k0 + kk];
#pragma unroll
        for (int a = 0; a < UJ; ++a) {
          const int j = j0 + JT * a;
          if (j < u) {
            const float* wr = w + kk * u4 + j;
            const float wi = wr[0], wf = wr[u], wc = wr[2 * u], wo = wr[3 * u];
#pragma unroll
            for (int i = 0; i < RJ; ++i) {
              acc[a][i][0] = fmaf(hv[i], wi, acc[a][i][0]);
              acc[a][i][1] = fmaf(hv[i], wf, acc[a][i][1]);
              acc[a][i][2] = fmaf(hv[i], wc, acc[a][i][2]);
              acc[a][i][3] = fmaf(hv[i], wo, acc[a][i][3]);
            }
          }
        }
      }
    }

#pragma unroll
    for (int i = 0; i < RJ; ++i) {
      const int row = g + G * i;
      const long long b = b0 + row;
      if (b >= p.B) continue;
      const long long o = b * p.T + t;
      const bool keep = mask_kept<M>(p.mask, o);
#pragma unroll
      for (int a = 0; a < UJ; ++a) {
        const int j = j0 + JT * a;
        if (j >= u) continue;
        const float hp = hc[row * u + j];
        float h = hp;
        if (keep) {
          const float* z = p.gx + o * u4;
          const float ig = rnn_sigmoid(z[j] + acc[a][i][0]);
          const float fg = rnn_sigmoid(z[u + j] + acc[a][i][1]);
          const float gg = rnn_tanh(z[2 * u + j] + acc[a][i][2]);
          const float og = rnn_sigmoid(z[3 * u + j] + acc[a][i][3]);
          c[a][i] = fg * c[a][i] + ig * gg;
          h = og * rnn_tanh(c[a][i]);
          if (p.gates) {
            float* gt = p.gates + o * u4;
            gt[j] = ig; gt[u + j] = fg; gt[2 * u + j] = gg; gt[3 * u + j] = og;
          }
        }
        if (p.gates) {
          p.c_seq[o * u + j] = c[a][i];
          p.h_prev[o * u + j] = hp;
        }
        if (p.seq) p.seq[o * u + j] = h;
        if (t == p.T - 1) {
          p.h_last[b * u + j] = h;
          p.c_last[b * u + j] = c[a][i];
        }
        hn[row * u + j] = h;
      }
    }
    __syncthreads();
    cur ^= 1;
  }
}

template <typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
lstm_bwd_kernel(const LstmBwdArgs p) {
  extern __shared__ float sm[];
  const int u = p.u, u4 = 4 * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
  const int j0 = threadIdx.x % JT, g = threadIdx.x / JT;
  const long long b0 = (long long)blockIdx.x * R;
  float* sUT = sm + 2 * R * u4;   // U^T slice: column c of U is row c of sUT, stride u + 1
  const int ld = u + 1;
  const bool resident = p.cs >= u4;

  for (int e = threadIdx.x; e < 2 * R * u4; e += RNN_THREADS) sm[e] = 0.f;
  if (resident)
    for (long long e = threadIdx.x; e < (long long)u * u4; e += RNN_THREADS)
      sUT[(e % u4) * ld + e / u4] = __ldg(p.U + e);
  __syncthreads();

  float dh[UJ][RJ], dc[UJ][RJ];
#pragma unroll
  for (int a = 0; a < UJ; ++a)
#pragma unroll
    for (int i = 0; i < RJ; ++i) dh[a][i] = dc[a][i] = 0.f;

  for (long long t = p.T - 1; t >= 0; --t) {
    float* sg = sm + (t & 1) * R * u4;
    bool keep[RJ];
#pragma unroll
    for (int i = 0; i < RJ; ++i) {
      const int row = g + G * i;
      const long long b = b0 + row;
      const bool valid = b < p.B;
      const long long o = b * p.T + t;
      keep[i] = valid && mask_kept<M>(p.mask, o);
#pragma unroll
      for (int a = 0; a < UJ; ++a) {
        const int j = j0 + JT * a;
        if (!valid || j >= u) continue;
        float d = dh[a][i], dcc = dc[a][i];
        if (p.g_seq) d += p.g_seq[o * u + j];
        if (t == p.T - 1) {
          if (p.g_h) d += p.g_h[b * u + j];
          if (p.g_c) dcc += p.g_c[b * u + j];
        }
        float di = 0.f, df = 0.f, dg = 0.f, dout = 0.f;
        if (keep[i]) {
          const float* gt = p.gates + o * u4;
          const float ig = gt[j], fg = gt[u + j], gg = gt[2 * u + j], og = gt[3 * u + j];
          const float cp = t > 0 ? p.c_seq[(o - 1) * u + j] : (p.c0 ? p.c0[b * u + j] : 0.f);
          const float tc = rnn_tanh(p.c_seq[o * u + j]);
          dout = d * tc * rnn_sigmoid_grad(og);
          const float dct = dcc + d * og * rnn_tanh_grad(tc);
          di = dct * gg * rnn_sigmoid_grad(ig);
          df = dct * cp * rnn_sigmoid_grad(fg);
          dg = dct * ig * rnn_tanh_grad(gg);
          dcc = dct * fg;
        }
        dh[a][i] = d;      // what a masked step passes through; a kept step replaces it with dz.U^T below
        dc[a][i] = dcc;
        float* dzr = p.dz + o * u4;
        dzr[j] = di; dzr[u + j] = df; dzr[2 * u + j] = dg; dzr[3 * u + j] = dout;
        float* sgr = sg + row * u4;
        sgr[j] = di; sgr[u + j] = df; sgr[2 * u + j] = dg; sgr[3 * u + j] = dout;
      }
    }
    __syncthreads();

    float acc[UJ][RJ];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) acc[a][i] = 0.f;
    for (int n0 = 0; n0 < u4; n0 += p.cs) {
      const int cn = min(p.cs, u4 - n0);
      if (!resident) {
        __syncthreads();
        for (long long e = threadIdx.x; e < (long long)cn * u; e += RNN_THREADS) {
          const long long k = e / cn, cc = e % cn;
          sUT[cc * ld + k] = __ldg(p.U + k * u4 + n0 + cc);
        }
        __syncthreads();
      }
      const float* w = resident ? sUT + (long long)n0 * ld : sUT;
      for (int cc = 0; cc < cn; ++cc) {
        float gv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) gv[i] = sg[(g + G * i) * u4 + n0 + cc];
#pragma unroll
        for (int a = 0; a < UJ; ++a) {
          const int j = j0 + JT * a;
          if (j < u) {
            const float wv = w[cc * ld + j];
#pragma unroll
            for (int i = 0; i < RJ; ++i) acc[a][i] = fmaf(gv[i], wv, acc[a][i]);
          }
        }
      }
    }
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i)
        if (keep[i]) dh[a][i] = acc[a][i];
  }

#pragma unroll
  for (int i = 0; i < RJ; ++i) {
    const long long b = b0 + g + G * i;
#pragma unroll
    for (int a = 0; a < UJ; ++a) {
      const int j = j0 + JT * a;
      if (b >= p.B || j >= u) continue;
      if (p.dh0) p.dh0[b * u + j] = dh[a][i];
      if (p.dc0) p.dc0[b * u + j] = dc[a][i];
    }
  }
}

template <typename M, int UJ, int RJ>
struct LstmFwdLaunch {
  static int run(const LstmFwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((lstm_fwd_kernel<M, UJ, RJ>), RNN_SMEM_MAX);
    lstm_fwd_kernel<M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
};

template <typename M, int UJ, int RJ>
struct LstmBwdLaunch {
  static int run(const LstmBwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((lstm_bwd_kernel<M, UJ, RJ>), RNN_SMEM_MAX);
    lstm_bwd_kernel<M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
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
  LstmFwdArgs a{gx, U, h0, c0, mask, B, T, units, tl.jt, 0, out_seq, h_last, c_last, gates, c_seq, h_prev};
  size_t smem;
  rnn_smem(2 * tl.rows * units, units, 4 * units, &a.ks, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  return rnn_dispatch<LstmFwdLaunch>("lstm_fwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
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
  LstmBwdArgs a{U, gates, c_seq, c0, mask, g_seq, g_h, g_c, B, T, units, tl.jt, 0, dz, dh0, dc0};
  size_t smem;
  rnn_smem(2 * tl.rows * 4 * units, 4 * units, units + 1, &a.cs, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  rc = rnn_dispatch<LstmBwdLaunch>("lstm_bwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
  if (rc || !dU) return rc;
  // dU = h_prev^T . dz: K6's backward of a linear layer whose output gradient is dz
  return tfrs_dense_bwd_f32(h_prev, U, dz, dz, nullptr, (long long)B * T, units, 4 * units, TFRS_ACT_LINEAR, nullptr, dU,
                            nullptr, ws, ws_bytes, stream);
}
