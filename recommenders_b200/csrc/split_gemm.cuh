// split_gemm.cuh -- the split-fp16 tensor-core GEMM (split_gemm.cu) behind the Cross (full-rank and low-rank) and Dense
// layers and tfrs_gemm_tc_f32:  C[M,N] = A'[M,K] . B'[N,K]^T,  ~2^-21 relative error.
#pragma once
#include "common.cuh"

namespace tfrs {
namespace tc {

// An operand: element (image row r, reduction index k) = transposed ? ptr[k * ld + r] : ptr[r * ld + k].
// amax_bits (nullable, device): max |element| as float bits when the caller already knows it; skips the statistics pass.
struct GemmOperand { const float* ptr; long long ld; bool transposed; const unsigned int* amax_bits = nullptr; };
enum { GEMM_EPI_PLAIN = 0, GEMM_EPI_DX = 1, GEMM_EPI_CROSS = 2, GEMM_EPI_DENSE = 3 };
// PLAIN: C = acc.   DX: C = acc + diag * e0 + e1.   CROSS: pv = acc + bias + diag * e1; prod = pv; C = e0 * pv + e1
// (ld0 == ld1 == ld_out); out_amax (nullable, device) receives max |C| as float bits.
// DENSE: z = acc + bias; C = act(z) (act = TFRS_ACT_*); prod = z when act is sigmoid (nullable).
// Every mode accumulates K > 1024 in chunks of 1024 (the tensor core's fp32 adder truncates, so one long chain drifts: a
// full-rank Cross at D = 4096 missed the 1e-5 bar), summed in fixed order before the epilogue; K <= 1024 is one launch.
struct GemmEpilogue { int mode; const float* e0; long long ld0; const float* e1; long long ld1; const float* bias; float diag; float* prod;
                      int act; unsigned int* out_amax = nullptr; };
// workspace of one gemm_tc call (the same for every epilogue)
size_t gemm_tc_workspace(long long M, long long N, long long K);
int gemm_tc(const GemmOperand& A, const GemmOperand& B, long long M, long long N, long long K, const GemmEpilogue& ep,
            float* out, long long ld_out, void* ws, size_t ws_bytes, cudaStream_t st);

}  // namespace tc
}  // namespace tfrs
