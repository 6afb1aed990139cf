// gru.cu -- K19: the recurrence of tf.keras.layers.GRU (reset_after=True, the TF2 default) as the reference's sequential
// retrieval tutorial builds its query tower (`Sequential([StringLookup, Embedding, GRU(32)])`).  The input projection
// gx = x.W + b_i is K6 (dense.cu) and comes in precomputed; this file owns the T-step recurrence, one launch each way.
//
//   Each CTA owns a tile of R batch rows for the whole sequence; rows are independent, so the only synchronisation is
//   __syncthreads.  Thread (j0, g) owns hidden units j = j0 + JT*a (a < UJ) of the tile rows g + G*i (i < RJ), with
//   JT = u rounded up to a power of two from 32 to 256, G = 256 / JT, UJ = ceil(u / JT) rounded up to a power of two
//   (1, 2, 4, 8: the kernel instances) and RJ = 8 / UJ, so R = G * RJ and R * u <= 2048: the tile shrinks as u grows,
//   and the two h buffers never pass 16 KB.
//   forward, per step: gr = h_{t-1}.U (+ b_r) as the fmaf chain over k ascending from +0.0f, the h tile and U read from
//     shared memory (U resident when it fits, otherwise streamed from L2 in k-slices every step); then the gate epilogue
//     writes h_t into the other h buffer.
//   backward, per step in reverse: the gate gradients of every owned pair, dgr staged in shared memory (two buffers, so
//     one barrier per step), then dh <- dh z + dgr.U^T as the fmaf chain over the 3u columns ascending, U^T staged like U.
//     The same C entry then runs K6's backward for dU = h_{t-1}^T . dgr and db_r = colsum(dgr).
//   A masked step does no arithmetic: the forward carries h, the backward passes dh through and writes zero rows.
#include "rnn.cuh"

namespace tfrs {

struct GruFwdArgs {
  const float* gx; const float* U; const float* br; const float* h0; const void* mask;
  long long B, T; int u, jt, ks;
  float* seq; float* h_last; float* gates; float* h_prev;
};

struct GruBwdArgs {
  const float* U; const float* gates; const float* h_prev; const void* mask; const float* g_seq; const float* g_last;
  long long B, T; int u, jt, cs;
  float* dgx; float* dgr; float* dh0;
};

template <typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
gru_fwd_kernel(const GruFwdArgs p) {
  extern __shared__ float sm[];
  const int u = p.u, u3 = 3 * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
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
    for (int e = threadIdx.x; e < u * u3; e += RNN_THREADS) sU[e] = __ldg(p.U + e);
  __syncthreads();

  int cur = 0;
  for (long long t = 0; t < p.T; ++t) {
    const float* hc = sm + cur * R * u;
    float* hn = sm + (cur ^ 1) * R * u;
    float acc[UJ][RJ][3];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) acc[a][i][0] = acc[a][i][1] = acc[a][i][2] = 0.f;

    for (int k0 = 0; k0 < u; k0 += p.ks) {
      const int kn = min(p.ks, u - k0);
      if (!resident) {
        __syncthreads();
        const float* src = p.U + (long long)k0 * u3;
        for (int e = threadIdx.x; e < kn * u3; e += RNN_THREADS) sU[e] = __ldg(src + e);
        __syncthreads();
      }
      const float* w = resident ? sU + (long long)k0 * u3 : sU;
      for (int kk = 0; kk < kn; ++kk) {
        float hv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) hv[i] = hc[(g + G * i) * u + k0 + kk];
#pragma unroll
        for (int a = 0; a < UJ; ++a) {
          const int j = j0 + JT * a;
          if (j < u) {
            const float wz = w[kk * u3 + j], wr = w[kk * u3 + u + j], wh = w[kk * u3 + 2 * u + j];
#pragma unroll
            for (int i = 0; i < RJ; ++i) {
              acc[a][i][0] = fmaf(hv[i], wz, acc[a][i][0]);
              acc[a][i][1] = fmaf(hv[i], wr, acc[a][i][1]);
              acc[a][i][2] = fmaf(hv[i], wh, acc[a][i][2]);
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
          const float* gxr = p.gx + o * u3;
          float gz = acc[a][i][0], gr = acc[a][i][1], gh = acc[a][i][2];
          if (p.br) { gz += __ldg(p.br + j); gr += __ldg(p.br + u + j); gh += __ldg(p.br + 2 * u + j); }
          const float z = rnn_sigmoid(gxr[j] + gz);
          const float r = rnn_sigmoid(gxr[u + j] + gr);
          const float hh = rnn_tanh(gxr[2 * u + j] + r * gh);
          h = z * hp + (1.f - z) * hh;
          if (p.gates) {
            float* gt = p.gates + o * 4 * u;
            gt[j] = z; gt[u + j] = r; gt[2 * u + j] = hh; gt[3 * u + j] = gh;
          }
        }
        if (p.h_prev) p.h_prev[o * u + j] = hp;
        if (p.seq) p.seq[o * u + j] = h;
        if (t == p.T - 1) p.h_last[b * u + j] = h;
        hn[row * u + j] = h;
      }
    }
    __syncthreads();
    cur ^= 1;
  }
}

template <typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
gru_bwd_kernel(const GruBwdArgs p) {
  extern __shared__ float sm[];
  const int u = p.u, u3 = 3 * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
  const int j0 = threadIdx.x % JT, g = threadIdx.x / JT;
  const long long b0 = (long long)blockIdx.x * R;
  float* sUT = sm + 2 * R * u3;   // U^T slice: column c of U is row c of sUT, stride u + 1
  const int ld = u + 1;
  const bool resident = p.cs >= u3;

  for (int e = threadIdx.x; e < 2 * R * u3; e += RNN_THREADS) sm[e] = 0.f;
  if (resident)
    for (long long e = threadIdx.x; e < (long long)u * u3; e += RNN_THREADS)
      sUT[(e % u3) * ld + e / u3] = __ldg(p.U + e);
  __syncthreads();

  float dh[UJ][RJ];
#pragma unroll
  for (int a = 0; a < UJ; ++a)
#pragma unroll
    for (int i = 0; i < RJ; ++i) dh[a][i] = 0.f;

  for (long long t = p.T - 1; t >= 0; --t) {
    float* sg = sm + (t & 1) * R * u3;
    float carry[UJ][RJ];
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
        carry[a][i] = dh[a][i];
        if (!valid || j >= u) continue;
        float d = dh[a][i];
        if (p.g_seq) d += p.g_seq[o * u + j];
        if (p.g_last && t == p.T - 1) d += p.g_last[b * u + j];
        float dz = 0.f, dr = 0.f, dhp = 0.f, dgh = 0.f;
        if (keep[i]) {
          const float* gt = p.gates + o * 4 * u;
          const float z = gt[j], r = gt[u + j], hh = gt[2 * u + j], grh = gt[3 * u + j];
          const float hp = p.h_prev[o * u + j];
          dz = d * (hp - hh) * rnn_sigmoid_grad(z);
          dhp = d * (1.f - z) * rnn_tanh_grad(hh);
          dr = dhp * grh * rnn_sigmoid_grad(r);
          dgh = dhp * r;
          carry[a][i] = d * z;
        } else {
          carry[a][i] = d;
        }
        float* gx = p.dgx + o * u3;
        float* gr = p.dgr + o * u3;
        gx[j] = dz; gx[u + j] = dr; gx[2 * u + j] = dhp;
        gr[j] = dz; gr[u + j] = dr; gr[2 * u + j] = dgh;
        sg[row * u3 + j] = dz; sg[row * u3 + u + j] = dr; sg[row * u3 + 2 * u + j] = dgh;
      }
    }
    __syncthreads();

    float acc[UJ][RJ];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) acc[a][i] = 0.f;
    for (int c0 = 0; c0 < u3; c0 += p.cs) {
      const int cn = min(p.cs, u3 - c0);
      if (!resident) {
        __syncthreads();
        for (long long e = threadIdx.x; e < (long long)cn * u; e += RNN_THREADS) {
          const long long k = e / cn, cc = e % cn;
          sUT[cc * ld + k] = __ldg(p.U + k * u3 + c0 + cc);
        }
        __syncthreads();
      }
      const float* w = resident ? sUT + (long long)c0 * ld : sUT;
      for (int cc = 0; cc < cn; ++cc) {
        float gv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) gv[i] = sg[(g + G * i) * u3 + c0 + cc];
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
      for (int i = 0; i < RJ; ++i) dh[a][i] = keep[i] ? carry[a][i] + acc[a][i] : carry[a][i];
  }

  if (p.dh0) {
#pragma unroll
    for (int i = 0; i < RJ; ++i) {
      const long long b = b0 + g + G * i;
#pragma unroll
      for (int a = 0; a < UJ; ++a) {
        const int j = j0 + JT * a;
        if (b < p.B && j < u) p.dh0[b * u + j] = dh[a][i];
      }
    }
  }
}

template <typename M, int UJ, int RJ>
struct GruFwdLaunch {
  static int run(const GruFwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((gru_fwd_kernel<M, UJ, RJ>), RNN_SMEM_MAX);
    gru_fwd_kernel<M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
};

template <typename M, int UJ, int RJ>
struct GruBwdLaunch {
  static int run(const GruBwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((gru_bwd_kernel<M, UJ, RJ>), RNN_SMEM_MAX);
    gru_bwd_kernel<M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
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
  GruFwdArgs a{gx, U, b_r, h0, mask, B, T, units, tl.jt, 0, out_seq, h_last, gates, h_prev};
  size_t smem;
  rnn_smem(2 * tl.rows * units, units, 3 * units, &a.ks, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  return rnn_dispatch<GruFwdLaunch>("gru_fwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
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
  GruBwdArgs a{U, gates, h_prev, mask, g_seq, g_last, B, T, units, tl.jt, 0, dgx, dgr, dh0};
  size_t smem;
  rnn_smem(2 * tl.rows * 3 * units, 3 * units, units + 1, &a.cs, &smem);
  const unsigned grid = (unsigned)ceil_div(B, tl.rows);
  rc = rnn_dispatch<GruBwdLaunch>("gru_bwd", mask_kind, tl.uj, a, grid, smem, (cudaStream_t)stream);
  if (rc || (!dU && !db_r)) return rc;
  // dU = h_prev^T . dgr, db_r = colsum(dgr): K6's backward of a linear layer whose output gradient is dgr
  return tfrs_dense_bwd_f32(h_prev, U, dgr, dgr, nullptr, n, units, 3 * units, TFRS_ACT_LINEAR, nullptr, dU, db_r, kws,
                            ws_bytes - (size_t)(kws - (unsigned char*)ws), stream);
}
