// cross_tc.cuh -- entry points of the tensor-core Cross backward GEMMs (cross_tc_bwd.cu), called from cross.cu.
#pragma once
#include "common.cuh"

namespace tfrs {
namespace tc {

size_t cross_tc_bwd_gemm_workspace(long long B, int D);
// dx = gp . W^T + diag * gp + dout (if dx != NULL);  dW = x^T . gp (if dW != NULL).  gp is dense [B,D]; x / dout / dx
// have row stride ld.
int cross_tc_bwd_gemms(const float* x, const float* W, const float* gp, const float* dout, long long B, int D, long long ld,
                       float diag, float* dx, float* dW, void* ws, size_t ws_bytes, cudaStream_t st);

// General split-fp16 tensor-core GEMM (cross_tc_bwd.cu):  C[M,N] = A'[M,K] . B'[N,K]^T,  ~2^-21 relative error.
// An operand: element (image row r, reduction index k) = transposed ? ptr[k * ld + r] : ptr[r * ld + k].
struct GemmOperand { const float* ptr; long long ld; bool transposed; };
enum { GEMM_EPI_PLAIN = 0, GEMM_EPI_DX = 1, GEMM_EPI_CROSS = 2, GEMM_EPI_DENSE = 3 };
// PLAIN: C = acc.   DX: C = acc + diag * e0 + e1.   CROSS: pv = acc + bias + diag * e1; prod = pv; C = e0 * pv + e1.
// DENSE: z = acc + bias; C = act(z) (act = TFRS_ACT_*); prod = z when act is sigmoid (nullable).  Any K (chunked above 1024).
struct GemmEpilogue { int mode; const float* e0; long long ld0; const float* e1; long long ld1; const float* bias; float diag; float* prod;
                      int act; };
size_t gemm_tc_workspace(long long M, long long N, long long K);
int gemm_tc(const GemmOperand& A, const GemmOperand& B, long long M, long long N, long long K, const GemmEpilogue& ep,
            float* out, long long ld_out, void* ws, size_t ws_bytes, cudaStream_t st);

}  // namespace tc
}  // namespace tfrs
