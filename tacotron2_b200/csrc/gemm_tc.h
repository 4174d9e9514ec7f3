// General fp32-grade GEMM / column sums of the training path on the tensor cores (gemm_tc.cu).
#pragma once
#include "model.h"

namespace t2 {

// row-major C (M x N, ldc) = op(A) . op(B) + beta C;  ta: A is stored (K x M, lda);  tb: B is stored (N x K, ldb).
// batch > 1: independent problems at element strides strideA / strideB / strideC (one set of operand scales).
// ws: the caller's scratch (operand scales, split-K partial tiles) of at least gemm_tc_ws_bytes(M, N, K, batch) bytes,
// 256-byte aligned; calls on one stream may share it.
// entry_rows (device, batch entries; the ragged log-mel path): entry b is computed exactly as the batch = 1 call over its
// first entry_rows[b] rows of op(A) (at most M): its own row scales, the K-split plan of gemm_tc(entry_rows[b], N, K,
// batch = 1) with its partial tiles added in the same order (inside the CTA, no partial buffer), and rows from
// entry_rows[b] on of C left unwritten.  Needs a K-contiguous op(A) (!ta), one op(B) for every entry (strideB = 0) and
// beta = 0; scratch: gemm_tc_ragged_ws_bytes(M, N, batch).
struct GemmTc {
  bool ta = false, tb = false;
  int M = 0, N = 0, K = 0;
  const float* A = nullptr; long lda = 0;
  const float* B = nullptr; long ldb = 0;
  float* C = nullptr; long ldc = 0;
  float beta = 0.f;
  int batch = 1; long strideA = 0, strideB = 0, strideC = 0;
  void* ws = nullptr; size_t ws_bytes = 0;
  const int* entry_rows = nullptr;
};
// sm_count plans the K splits; calls without a model (mel_spectrogram, the self-tests) plan for kGemmTcSms
constexpr int kGemmTcSms = 132;
size_t gemm_tc_ws_bytes(int M, int N, int K, int batch = 1);
size_t gemm_tc_ragged_ws_bytes(int M, int N, int batch);
int gemm_tc(int sm_count, cudaStream_t s, const GemmTc& g);
int gemm_tc_rm(int sm_count, cudaStream_t s, void* ws, size_t ws_bytes, bool ta, bool tb, int M, int N, int K, const float* A,
               long lda, const float* B, long ldb, float* C, long ldc, float beta);
// out[c] = sum over `rows` rows of X[r * ld + c]; ws: at least colsum_ws_bytes(rows, cols) bytes
size_t colsum_ws_bytes(long rows, int cols);
int colsum_f32(cudaStream_t s, void* ws, size_t ws_bytes, const float* X, long ld, long rows, int cols, float* out);

}  // namespace t2
