// rnn.cuh -- the recurrence kernels of K19 (gru.cu) and K20 (lstm.cu): one forward and one reverse kernel, templated on
// the cell, with the gate arithmetic, the plan of a CTA's (row, unit) pairs, the shared-memory budget and the choice of
// kernel instance.  The input projection gx = x.W + b is K6 (dense.cu) and comes in precomputed; these kernels own the
// T-step recurrence, one launch each way.  The gate derivatives are taken from the saved gate OUTPUTS, as TF's
// SigmoidGrad / TanhGrad do.
//
//   Each CTA owns a tile of R batch rows for the whole sequence; rows are independent, so the only synchronisation is
//   __syncthreads.  Thread (j0, g) owns hidden units j = j0 + JT*a (a < UJ) of the tile rows g + G*i (i < RJ) at every
//   step (rnn_tile), so h is double-buffered in shared memory (R * u <= 2048: at most 16 KB) and the cell's own state
//   (LSTM's c) never leaves registers.  U is [u, NG*u] for NG gates.
//   forward, per step: the NG fmaf chains h_{t-1}.U (one per gate column) over k ascending from +0.0f, the h tile and U
//     read from shared memory (U resident when it fits, otherwise streamed from L2 in k-slices every step); then the
//     cell's gate epilogue adds gx and writes h_t into the other h buffer.
//   backward, per step in reverse: the cell's gate gradients of every owned pair go to HBM and to shared memory (two
//     buffers, so one barrier per step), then the fmaf chain dgates.U^T over the NG*u columns ascending, U^T staged
//     transposed like U, and the cell combines it with the carried dh.
//   A masked step does no arithmetic: the forward carries h (and the cell's state), the backward passes dh through
//   and the cell writes zero gradient rows.
//
// A cell (GruCell, LstmCell) supplies NG, its per-pair register State, its FwdArgs / BwdArgs (derived from RnnFwdArgs
// / RnnBwdArgs) and these hooks, all inlined:
//   fwd_init(p, s, b, j)                   the state before step 0
//   fwd_gates(p, s, acc, o, j, hp) -> h_t  a kept step's gate epilogue from the chains acc[NG] and h_{t-1} = hp
//   fwd_save(p, s, o, j, hp)               what every step saves for the backward
//   fwd_last(p, s, bj)                     the final state beyond h_T
//   bwd_gates(p, s, d, keep, b, o, j, t, sgr) -> carry
//                                          the gate gradients for d = dh_t (+ the step's output gradient): to HBM and
//                                          to the row sgr (gate q of unit j at q*u + j); zero on a masked step
//   bwd_dh(keep, dh, acc)                  dh_{t-1} from the carry dh and the chain acc = dgates.U^T, in place
//   bwd_initial(p)                         whether the call asks for any initial-state gradient
//   bwd_last(p, s, bj)                     the initial-state gradients beyond dh0
// The hooks keep the parent kernels' operation order; forms that changed the compiled code of either cell (a
// shared dgates store, the combine as a return value) stay in the cells.
#pragma once
#include <utility>

#include "dense.cuh"

namespace tfrs {

// f(q) for the gates q = 0 .. N-1 (std::integral_constant), written out as straight-line code.  A loop over the gate
// count, even one unrolled later, changes how the compiler schedules the forward's chains: with one, GRU's (1, 8)
// instance grew from 2856 to 3080 instructions and its forward ran 10% slower at u = 128 and 256 (H100 SXM, 700 W).
template <typename F, int... Q>
__device__ __forceinline__ void rnn_gates(F&& f, std::integer_sequence<int, Q...>) {
  (f(std::integral_constant<int, Q>{}), ...);
}
template <int N, typename F>
__device__ __forceinline__ void rnn_gates(F&& f) {
  rnn_gates(f, std::make_integer_sequence<int, N>{});
}

// 1 / (1 + expf(-x)): the Dense layer's sigmoid
__device__ __forceinline__ float rnn_sigmoid(float x) { return dense_act(TFRS_ACT_SIGMOID, x); }
__device__ __forceinline__ float rnn_tanh(float x) { return tanhf(x); }
// sigmoid'(x) = s (1 - s) and tanh'(x) = 1 - y^2 from s = sigmoid(x), y = tanh(x)
__device__ __forceinline__ float rnn_sigmoid_grad(float s) { return s * (1.f - s); }
__device__ __forceinline__ float rnn_tanh_grad(float y) { return 1.f - y * y; }

constexpr int RNN_THREADS = 256;
constexpr int RNN_PAIRS = 8;                  // (row, unit) pairs per thread: R * JT = RNN_THREADS * RNN_PAIRS / UJ
constexpr int RNN_SMEM_MAX = 227 * 1024;      // sm_90 opt-in dynamic shared memory per block
constexpr int RNN_SLICE_BYTES = 64 * 1024;    // a streamed slice of U (or U^T) when the whole matrix does not fit

// Thread (j0, g) of a CTA owns hidden units j = j0 + JT*a (a < UJ) of the tile rows g + G*i (i < RJ).
struct RnnTile {
  int jt, g, uj, rj, rows;
};

static inline RnnTile rnn_tile(int u) {
  RnnTile t;
  t.jt = 32;   // a power of two, so that the G = RNN_THREADS / JT row groups use every thread and no two alias a row
  while (t.jt < u && t.jt < RNN_THREADS) t.jt *= 2;
  t.g = RNN_THREADS / t.jt;
  t.uj = 1;    // a power of two too, so that RJ = RNN_PAIRS / UJ is exact and names a kernel instance (rnn_tiles)
  while (t.uj * t.jt < u) t.uj *= 2;
  t.rj = RNN_PAIRS / t.uj;
  t.rows = t.g * t.rj;
  return t;
}

// shared memory of one CTA: the fixed part plus a weight matrix of `rows_total` rows of `per` floats, whole when it
// fits in the 227 KB, otherwise in slices of RNN_SLICE_BYTES (*slice_rows rows)
static inline void rnn_smem(int fixed_floats, int rows_total, int per, int* slice_rows, size_t* bytes) {
  const size_t fixed = (size_t)fixed_floats * 4, whole = (size_t)rows_total * per * 4;
  if (fixed + whole <= (size_t)RNN_SMEM_MAX) {
    *slice_rows = rows_total;
    *bytes = fixed + whole;
    return;
  }
  int s = RNN_SLICE_BYTES / (per * 4);
  *slice_rows = s < 1 ? 1 : s;
  *bytes = fixed + (size_t)*slice_rows * per * 4;
}

// what the shared kernels read and write; the cells' argument structs add their own fields
struct RnnFwdArgs {
  const float* gx; const float* U; const float* h0; const void* mask;
  long long B, T; int u, jt, ks;
  float* seq; float* h_last;
};

struct RnnBwdArgs {
  const float* U; const void* mask; const float* g_seq;
  long long B, T; int u, jt, cs;
  float* dh0;
};

template <typename Cell, typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
rnn_fwd_kernel(const typename Cell::FwdArgs p) {
  constexpr int NG = Cell::NG;
  extern __shared__ float sm[];
  const int u = p.u, nu = NG * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
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
    for (int e = threadIdx.x; e < u * nu; e += RNN_THREADS) sU[e] = __ldg(p.U + e);
  typename Cell::State s[UJ][RJ];
#pragma unroll
  for (int i = 0; i < RJ; ++i)
#pragma unroll
    for (int a = 0; a < UJ; ++a) Cell::fwd_init(p, s[a][i], b0 + g + G * i, j0 + JT * a);
  __syncthreads();

  int cur = 0;
  for (long long t = 0; t < p.T; ++t) {
    const float* hc = sm + cur * R * u;
    float* hn = sm + (cur ^ 1) * R * u;
    float acc[UJ][RJ][NG];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) rnn_gates<NG>([&](auto q) { acc[a][i][q] = 0.f; });

    for (int k0 = 0; k0 < u; k0 += p.ks) {
      const int kn = min(p.ks, u - k0);
      if (!resident) {
        __syncthreads();
        const float* src = p.U + (long long)k0 * nu;
        for (int e = threadIdx.x; e < kn * nu; e += RNN_THREADS) sU[e] = __ldg(src + e);
        __syncthreads();
      }
      const float* w = resident ? sU + (long long)k0 * nu : sU;
      for (int kk = 0; kk < kn; ++kk) {
        float hv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) hv[i] = hc[(g + G * i) * u + k0 + kk];
#pragma unroll
        for (int a = 0; a < UJ; ++a) {
          const int j = j0 + JT * a;
          if (j < u) {
            const float* wr = w + kk * nu + j;
            float wv[NG];
            rnn_gates<NG>([&](auto q) { wv[q] = wr[q * u]; });
#pragma unroll
            for (int i = 0; i < RJ; ++i) rnn_gates<NG>([&](auto q) { acc[a][i][q] = fmaf(hv[i], wv[q], acc[a][i][q]); });
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
        if (keep) h = Cell::fwd_gates(p, s[a][i], acc[a][i], o, j, hp);
        Cell::fwd_save(p, s[a][i], o, j, hp);
        if (p.seq) p.seq[o * u + j] = h;
        if (t == p.T - 1) {
          p.h_last[b * u + j] = h;
          Cell::fwd_last(p, s[a][i], b * u + j);
        }
        hn[row * u + j] = h;
      }
    }
    __syncthreads();
    cur ^= 1;
  }
}

template <typename Cell, typename M, int UJ, int RJ>
__global__ void __launch_bounds__(RNN_THREADS, 2)
rnn_bwd_kernel(const typename Cell::BwdArgs p) {
  constexpr int NG = Cell::NG;
  extern __shared__ float sm[];
  const int u = p.u, nu = NG * u, JT = p.jt, G = RNN_THREADS / JT, R = G * RJ;
  const int j0 = threadIdx.x % JT, g = threadIdx.x / JT;
  const long long b0 = (long long)blockIdx.x * R;
  float* sUT = sm + 2 * R * nu;   // U^T slice: column c of U is row c of sUT, stride u + 1
  const int ld = u + 1;
  const bool resident = p.cs >= nu;

  for (int e = threadIdx.x; e < 2 * R * nu; e += RNN_THREADS) sm[e] = 0.f;
  if (resident)
    for (long long e = threadIdx.x; e < (long long)u * nu; e += RNN_THREADS)
      sUT[(e % nu) * ld + e / nu] = __ldg(p.U + e);
  __syncthreads();

  float dh[UJ][RJ];
  typename Cell::State s[UJ][RJ];
#pragma unroll
  for (int a = 0; a < UJ; ++a)
#pragma unroll
    for (int i = 0; i < RJ; ++i) {
      dh[a][i] = 0.f;
      s[a][i] = {};
    }

  for (long long t = p.T - 1; t >= 0; --t) {
    float* sg = sm + (t & 1) * R * nu;
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
        float d = dh[a][i];
        if (p.g_seq) d += p.g_seq[o * u + j];
        dh[a][i] = Cell::bwd_gates(p, s[a][i], d, keep[i], b, o, j, t, sg + row * nu);
      }
    }
    __syncthreads();

    float acc[UJ][RJ];
#pragma unroll
    for (int a = 0; a < UJ; ++a)
#pragma unroll
      for (int i = 0; i < RJ; ++i) acc[a][i] = 0.f;
    for (int c0 = 0; c0 < nu; c0 += p.cs) {
      const int cn = min(p.cs, nu - c0);
      if (!resident) {
        __syncthreads();
        for (long long e = threadIdx.x; e < (long long)cn * u; e += RNN_THREADS) {
          const long long k = e / cn, cc = e % cn;
          sUT[cc * ld + k] = __ldg(p.U + k * nu + c0 + cc);
        }
        __syncthreads();
      }
      const float* w = resident ? sUT + (long long)c0 * ld : sUT;
      for (int cc = 0; cc < cn; ++cc) {
        float gv[RJ];
#pragma unroll
        for (int i = 0; i < RJ; ++i) gv[i] = sg[(g + G * i) * nu + c0 + cc];
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
      for (int i = 0; i < RJ; ++i) Cell::bwd_dh(keep[i], dh[a][i], acc[a][i]);
  }

  if (Cell::bwd_initial(p)) {
#pragma unroll
    for (int i = 0; i < RJ; ++i) {
      const long long b = b0 + g + G * i;
#pragma unroll
      for (int a = 0; a < UJ; ++a) {
        const int j = j0 + JT * a;
        if (b < p.B && j < u) {
          if (p.dh0) p.dh0[b * u + j] = dh[a][i];
          Cell::bwd_last(p, s[a][i], b * u + j);
        }
      }
    }
  }
}

// the forward or the reverse kernel of the cell, by the argument type, at the tile (UJ, RJ) and mask element type M
template <typename Cell, typename M, int UJ, int RJ>
struct RnnLaunch {
  static int run(const typename Cell::FwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((rnn_fwd_kernel<Cell, M, UJ, RJ>), RNN_SMEM_MAX);
    rnn_fwd_kernel<Cell, M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  static int run(const typename Cell::BwdArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
    TFRS_DYN_SMEM((rnn_bwd_kernel<Cell, M, UJ, RJ>), RNN_SMEM_MAX);
    rnn_bwd_kernel<Cell, M, UJ, RJ><<<grid, RNN_THREADS, smem, st>>>(a);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
};

// RnnLaunch<Cell, M, UJ, RJ>::run for the tile of u (UJ units per thread, RJ = RNN_PAIRS / UJ rows)
template <typename Cell, typename M, typename A>
static int rnn_tiles(const char* what, int uj, const A& a, unsigned grid, size_t smem, cudaStream_t st) {
  switch (uj) {
    case 1: return RnnLaunch<Cell, M, 1, 8>::run(a, grid, smem, st);
    case 2: return RnnLaunch<Cell, M, 2, 4>::run(a, grid, smem, st);
    case 4: return RnnLaunch<Cell, M, 4, 2>::run(a, grid, smem, st);
    case 8: return RnnLaunch<Cell, M, 8, 1>::run(a, grid, smem, st);
  }
  set_error("%s: no kernel instance for %d units per thread", what, uj);
  return TFRS_ERR_INVALID_ARG;
}

// ... and for the mask's element type
template <typename Cell, typename A>
static int rnn_dispatch(const char* what, int mask_kind, int uj, const A& a, unsigned grid, size_t smem,
                        cudaStream_t st) {
  return mask_dispatch(a.mask, mask_kind,
                       [&](auto m) { return rnn_tiles<Cell, decltype(m)>(what, uj, a, grid, smem, st); });
}

static inline int rnn_check(const char* what, int64_t B, int64_t T, int u, int max_units, const void* mask,
                            int mask_kind) {
  TFRS_CHECK_ARG(B >= 0 && B < (1ll << 31) && T >= 1 && T < (1ll << 31) && u >= 1 && u <= max_units,
                 "%s: bad shape B=%lld T=%lld units=%d (1 <= units <= %d, T >= 1)", what, (long long)B, (long long)T, u,
                 max_units);
  TFRS_CHECK_MASK(what, mask, mask_kind);
  return TFRS_OK;
}

}  // namespace tfrs
