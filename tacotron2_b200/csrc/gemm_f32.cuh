// fp32 SIMT GEMM  C = epilogue( sum_s A_s (M x K_s) * W_s (N x K_s)^T )  -- the stepwise decoder (T2_IMPL_STEPWISE), the
// decoders' processed memory, the prenet forward / backward and the encoder's LSTM input projection behind the training
// conv stack.  Up to 3 K-segments avoid materialising torch.cat() of the reference (model.py:352, 366-367, 373-374).
#pragma once
#include "common.cuh"

namespace t2 {

struct GemmSeg {
  const float* A; long lda;   // (M, K) row-major
  const float* W; long ldw;   // (N, K) row-major
  int K;                      // multiple of 16
};

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2 };

struct GemmArgs {
  GemmSeg seg[3];
  int nseg = 1;
  int M = 0, N = 0;
  float* C = nullptr; long ldc = 0;
  const float* bias = nullptr;    // (N) added to the accumulator
  int act = ACT_NONE;
  // dropout on the output: explicit keep mask (M, N) uint8 or Philox(seed, site); p = drop prob
  const uint8_t* keep = nullptr; long ldkeep = 0;
  int philox = 0; uint64_t seed = 0; uint32_t site = 0; float p_drop = 0.f;
  const uint64_t* row_seeds = nullptr;   // (M) or null: Philox(row_seeds[m], site), element n instead of seed, m * N + n
  const int* skip_flag = nullptr;    // device flag: when *skip_flag != 0 the kernel is a no-op
};

int gemm_f32(const GemmArgs& a, cudaStream_t s);

}  // namespace t2
