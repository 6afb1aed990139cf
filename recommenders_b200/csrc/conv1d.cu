// conv1d.cu -- K27: the 1-D convolution of layers.Conv1D (tf.keras.layers.Conv1D, channels_last, groups = 1) over x [B, T, C]
// with W [k, C, F] and stride s, dilation d, left pad p:
//   y[b, t, n] = act(bias[n] + sum_j sum_c x[b, t s + j d - p, c] W[j, c, n]),  positions outside [0, T) read as 0,
// i.e. the Dense layer (K6) on the im2col matrix col [B T_out, k C] (split_gemm.cuh WindowSrc) with W viewed as [k C, F].
//   tensor cores (K6's rule on (B T_out, k C, F)): K6's split-fp16 GEMM and DENSE epilogue, with the A image gathered from x
//     window by window (cx_window_image_kernel, split_gemm.cu), so col is never formed;
//   otherwise: col is gathered into the workspace (one launch) and K6's exact CUDA-core forward / backward run on it.
//   bwd: dz = dy act'(y) and dbias = colsum(dz) as K6; dW = col^T . dz (on tensor cores the transposed window gather is the A
//   image, the reduction over B T_out chunked by 1024 and summed in fixed order); dcol = dz . W^T into the workspace; then
//   dx = col2im(dcol): dx[b, t, c] = the sum over j ascending of dcol[(b, t_out), j C + c] for the t_out with
//   t_out s + j d - p = t.  No float atomics: bitwise reproducible.
#include "split_gemm.cuh"
#include "dense.cuh"

namespace tfrs {

// col [M, kC] = the im2col matrix of `win` (M = B T_out, kC = k C), one element per thread
__global__ void __launch_bounds__(256)
conv1d_im2col_kernel(const tc::WindowSrc win, long long M, int kC, float* __restrict__ col) {
  const long long total = M * kC;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    const long long r = e / kC;
    col[e] = win.at(r, e - r * kC);
  }
}

// dx[b, t, c] = sum over j = 0 .. k-1 (ascending, from +0.0f) of dcol[b T_out + t_out, j C + c] where t + p - j d = t_out s,
// 0 <= t_out < T_out; one thread per element of dx
__global__ void __launch_bounds__(256)
conv1d_col2im_kernel(const float* __restrict__ dcol, long long B, int T, int C, int T_out, int k, int stride, int dilation, int pad,
                     float* __restrict__ dx) {
  const long long total = B * T * (long long)C;
  const long long kC = (long long)k * C;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    const long long bt = e / C; const int c = (int)(e - bt * C);
    const long long b = bt / T; const int t = (int)(bt - b * T);
    float acc = 0.f;
    for (int j = 0; j < k; ++j) {
      const int u = t + pad - j * dilation;
      if (u < 0) break;   // u falls as j grows
      const int to = u / stride;
      if (to * stride == u && to < T_out) acc += __ldg(dcol + (b * T_out + to) * kC + (long long)j * C + c);
    }
    dx[e] = acc;
  }
}

struct Conv1dShape { long long B, M; int T, C, k, F, kC, stride, dilation, pad, T_out; };

static size_t conv1d_fwd_ws(long long M, int kC, int F) {
  if (M <= 0) return 0;
  return dense_tc(M, kC, F) ? tc::gemm_tc_workspace(M, F, kC) : (size_t)M * kC * 4;
}

static size_t conv1d_bwd_ws(long long M, int kC, int F) {
  if (M <= 0) return 256;
  const size_t dcol = align_up((size_t)M * kC * 4, 1024);
  if (dense_tc(M, kC, F)) {
    const size_t a = tc::gemm_tc_workspace(M, kC, F), b = tc::gemm_tc_workspace(kC, F, M);
    return dcol + align_up((size_t)M * F * 4, 1024) + align_up(dense_colsum_bytes(F), 1024) + (a > b ? a : b);
  }
  return dcol + align_up((size_t)M * kC * 4, 1024) + tfrs_dense_bwd_workspace_bytes(M, kC, F);
}

static int conv1d_check(const char* what, int64_t B, int T, int C, int k, int F, int stride, int dilation, int pad, int T_out,
                        int activation, Conv1dShape& sh) {
  TFRS_CHECK_ARG(B >= 0 && T > 0 && C > 0 && k > 0 && F > 0 && stride > 0 && dilation > 0 && pad >= 0 && T_out > 0,
                 "%s: bad shape B=%lld T=%d C=%d k=%d filters=%d stride=%d dilation=%d pad=%d T_out=%d", what, (long long)B, T, C,
                 k, F, stride, dilation, pad, T_out);
  TFRS_CHECK_ARG((long long)k * C < (1ll << 31) && (long long)(T_out - 1) * stride + (long long)(k - 1) * dilation < (1ll << 31),
                 "%s: k * C or the receptive field is too large", what);
  TFRS_CHECK_ARG(B * T_out < (1ll << 31), "%s: B * T_out = %lld is too large", what, (long long)B * T_out);
  TFRS_CHECK_ARG(activation >= TFRS_ACT_LINEAR && activation <= TFRS_ACT_SIGMOID, "%s: unknown activation %d", what, activation);
  sh = Conv1dShape{B, B * T_out, T, C, k, F, k * C, stride, dilation, pad, T_out};
  return TFRS_OK;
}

static int conv1d_im2col(const tc::WindowSrc& win, long long M, int kC, float* col, cudaStream_t st) {
  conv1d_im2col_kernel<<<elementwise_grid(M * kC), 256, 0, st>>>(win, M, kC, col);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_conv1d_fwd_workspace_bytes(int64_t B, int T_out, int C, int k, int F) {
  if (B <= 0 || T_out <= 0 || C <= 0 || k <= 0 || F <= 0) return 0;
  return conv1d_fwd_ws(B * T_out, k * C, F);
}

extern "C" int tfrs_conv1d_fwd_f32(const float* x, const float* W, const float* bias, int64_t B, int T, int C, int k, int F, int stride,
                                   int dilation, int pad, int T_out, int activation, float* y, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x && W && y, "conv1d_fwd: NULL pointer");
  Conv1dShape sh;
  int rc = conv1d_check("conv1d_fwd", B, T, C, k, F, stride, dilation, pad, T_out, activation, sh);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  if (!ws || ws_bytes < conv1d_fwd_ws(sh.M, sh.kC, F)) { set_error("conv1d_fwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "conv1d_fwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const tc::WindowSrc win{x, T, C, T_out, stride, dilation, pad};
  if (dense_tc(sh.M, sh.kC, F)) {   // B operand: image row = filter n, reduction index kk: W[kk * F + n], as K6
    const tc::GemmEpilogue ep{tc::GEMM_EPI_DENSE, nullptr, 0, nullptr, 0, bias, 0.f, nullptr, activation};
    return tc::gemm_tc(tc::GemmOperand{nullptr, 0, false, nullptr, &win}, tc::GemmOperand{W, F, true}, sh.M, F, sh.kC, ep, y, F,
                       ws, ws_bytes, st);
  }
  float* col = (float*)ws;
  rc = conv1d_im2col(win, sh.M, sh.kC, col, st);
  if (rc) return rc;
  return tfrs_dense_fwd_f32(col, W, bias, sh.M, sh.kC, F, activation, y, nullptr, nullptr, 0, stream);
}

extern "C" size_t tfrs_conv1d_bwd_workspace_bytes(int64_t B, int T_out, int C, int k, int F) {
  if (B <= 0 || T_out <= 0 || C <= 0 || k <= 0 || F <= 0) return 256;
  return conv1d_bwd_ws(B * T_out, k * C, F);
}

extern "C" int tfrs_conv1d_bwd_f32(const float* x, const float* W, const float* y, const float* dy, int64_t B, int T, int C, int k,
                                   int F, int stride, int dilation, int pad, int T_out, int activation, float* dx, float* dW,
                                   float* dbias, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x && W && y && dy, "conv1d_bwd: NULL pointer");
  Conv1dShape sh;
  int rc = conv1d_check("conv1d_bwd", B, T, C, k, F, stride, dilation, pad, T_out, activation, sh);
  if (rc) return rc;
  TFRS_CHECK_ARG(B > 0, "conv1d_bwd: empty batch");
  if (!ws || ws_bytes < conv1d_bwd_ws(sh.M, sh.kC, F)) { set_error("conv1d_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "conv1d_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const tc::WindowSrc win{x, T, C, T_out, stride, dilation, pad};
  unsigned char* w = (unsigned char*)ws;
  float* dcol = (float*)w; w += align_up((size_t)sh.M * sh.kC * 4, 1024);
  if (dense_tc(sh.M, sh.kC, F)) {
    float* dz = (float*)w; w += align_up((size_t)sh.M * F * 4, 1024);
    double* colpart = (double*)w; w += align_up(dense_colsum_bytes(F), 1024);
    const size_t gws = ws_bytes - (size_t)(w - (unsigned char*)ws);
    rc = dense_dz(y, dy, nullptr, sh.M * F, activation, dz, st);
    if (rc) return rc;
    const tc::GemmEpilogue plain{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr, 0};
    if (dx) {   // dcol[r, kk] = sum_n dz[r, n] W[kk, n]
      rc = tc::gemm_tc(tc::GemmOperand{dz, F, false}, tc::GemmOperand{W, F, false}, sh.M, sh.kC, F, plain, dcol, sh.kC, w, gws, st);
      if (rc) return rc;
    }
    if (dW) {   // dW[kk, n] = sum_r col[r, kk] dz[r, n]
      rc = tc::gemm_tc(tc::GemmOperand{nullptr, 0, true, nullptr, &win}, tc::GemmOperand{dz, F, true}, sh.kC, F, sh.M, plain, dW, F,
                       w, gws, st);
      if (rc) return rc;
    }
    if (dbias) {
      rc = dense_colsum(dz, sh.M, F, colpart, dbias, st);
      if (rc) return rc;
    }
  } else {
    float* col = (float*)w; w += align_up((size_t)sh.M * sh.kC * 4, 1024);
    rc = conv1d_im2col(win, sh.M, sh.kC, col, st);
    if (rc) return rc;
    rc = tfrs_dense_bwd_f32(col, W, y, dy, nullptr, sh.M, sh.kC, F, activation, dx ? dcol : nullptr, dW, dbias, w,
                            ws_bytes - (size_t)(w - (unsigned char*)ws), stream);
    if (rc) return rc;
  }
  if (dx) {
    conv1d_col2im_kernel<<<elementwise_grid(B * T * (long long)C), 256, 0, st>>>(dcol, B, T, C, T_out, k, stride, dilation, pad, dx);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}
