// Tensor-core conv1d / GEMM for the Encoder (model.py:157-167, 174-175), the BiLSTM input projection
// (model.py:169-171) and the Postnet (model.py:112-146): the split-fp16 implicit GEMM of wg_gemm.cuh with its conv
// epilogue (EPI_CONV).  This file holds the operand formats and the host entry points.
//
//   out[(b,t), n] = epilogue( sum_{tap, ci} W[n][tap][ci] * x[(b, t + tap - pad), ci] )
//
// * Activations live in "k8 planes": for every group of 8 channels, a hi and a lo plane of
//   [rows][8] fp16 (16 bytes per row).  Rows are the sequences with 2 zero rows before and after each
//   (+2 guard rows at both ends of the plane), so a 128-row output tile needs input rows [m0-2, m0+130):
//   ONE contiguous 2112-byte bulk copy per plane, and the 5 taps of a conv are the SAME shared-memory
//   tile addressed with the descriptor start shifted by tap*16 bytes -- no im2col, 5x reuse from SMEM.
//   (K-major no-swizzle canonical layout with LBO = 2112 between k8 groups, SBO = 128 between 8-row groups.)
// * Weights are packed per (n-tile, 64-channel chunk, tap) as [hi | lo] SWIZZLE_128B planes of n-tile rows x 64
//   channels, the order in which the GEMM streams its weight stages.
// * fp32-grade: hi*hi + lo*hi + hi*lo, 3 MMAs (M=64 per warpgroup, N=n_tile, K=16) per 16 channels, fp32 in registers.
// * Epilogue: folded BatchNorm scale/shift (+bias), ReLU / tanh, and either the next layer's planes,
//   fp32 rows (LSTM gate pre-activations) or the final (B, 80, T) tensor with the residual (model.py:511/524).
#include <stdlib.h>
#include <string.h>

#include "conv_tc.h"
#include "wg_gemm.cuh"

namespace t2 {
namespace {

// ---- layout conversion kernels ---------------------------------------------------------------------
// fp32 channels-last rows (B, T, C) [batch stride] -> k8 planes with sequence padding; frames t >= len
// and channels >= C are zero; every row of every plane (incl. guards) is written.
__global__ void rows_to_planes_kernel(const float* __restrict__ x, long batch_stride, int C, int c_pad,
                                      const int32_t* __restrict__ len, int B, int T, __half* __restrict__ planes,
                                      long plane_rows, const float* __restrict__ in_scale) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;     // plane row (incl. 2 guard rows)
  const int g = blockIdx.y;
  if (row >= plane_rows) return;
  const long prow = row - 2;
  const int span = T + 4;
  int b = -1, t = -1;
  if (prow >= 0) { b = (int)(prow / span); t = (int)(prow - (long)b * span) - 2; }
  const bool valid = b >= 0 && b < B && t >= 0 && t < T && (len == nullptr || t < len[b]);
  const float mul = in_scale ? *in_scale : 1.f;       // power-of-two pre-scale (gradients do not fit fp16 otherwise)
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    v[i] = (valid && c < C) ? x[(long)b * batch_stride + (long)t * C + c] * mul : 0.f;
  }
  store8<3>(planes, plane_rows, g, row, v);
}

// embedding gather straight into planes (model.py:503 / 518); symbols at t >= len[b] are not read, their rows are zero
__global__ void embed_to_planes_kernel(const int64_t* __restrict__ text, const float* __restrict__ emb, int n_symbols,
                                       const int32_t* __restrict__ len, int B, int T, __half* __restrict__ planes,
                                       long plane_rows) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y;
  if (row >= plane_rows) return;
  const long prow = row - 2;
  const int span = T + 4;
  int b = -1, t = -1;
  if (prow >= 0) { b = (int)(prow / span); t = (int)(prow - (long)b * span) - 2; }
  const bool valid = b >= 0 && b < B && t >= 0 && t < T && (len == nullptr || t < len[b]);
  long id = 0;
  if (valid) { id = text[(long)b * T + t]; id = id < 0 ? 0 : (id >= n_symbols ? n_symbols - 1 : id); }
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = valid ? emb[id * kEnc + g * 8 + i] : 0.f;
  store8<3>(planes, plane_rows, g, row, v);
}

// W (cout, cin, taps) fp32 [or (cout, cin) when taps == 1] -> per (n-tile, chunk, tap) [hi | lo] SWIZZLE_128B
// planes of NT rows x 64 channels; rows >= cout and channels >= cin are zero.
__global__ void pack_conv_w_kernel(const float* __restrict__ w, int cout, int cin, int taps, int nt_rows,
                                   int nchunks, uint8_t* __restrict__ img) {
  const int tap = blockIdx.x % taps, c = (blockIdx.x / taps) % nchunks, nt = blockIdx.x / (taps * nchunks);
  __half* hi = reinterpret_cast<__half*>(img + (size_t)blockIdx.x * nt_rows * 256);
  __half* lo = hi + nt_rows * 64;
  for (int i = threadIdx.x; i < nt_rows * 64; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    const int n = nt * nt_rows + r, ci = c * 64 + k;
    const float v = (n < cout && ci < cin) ? w[((long)n * cin + ci) * taps + tap] : 0.f;
    __half h, l;
    split_fp16(v, h, l);
    const uint32_t e = img_elem_offset(r, k);
    hi[e] = h; lo[e] = l;
  }
}

__global__ void fold_bn_bias_kernel(const float* cbias, const float* g, const float* b, const float* mean,
                                    const float* var, float eps, float* scale, float* shift, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (g == nullptr) { scale[c] = 1.f; shift[c] = cbias ? cbias[c] : 0.f; return; }
  const float s = g[c] / sqrtf(var[c] + eps);
  scale[c] = s;
  shift[c] = b[c] + ((cbias ? cbias[c] : 0.f) - mean[c]) * s;
}

}  // namespace

// ---- host API -------------------------------------------------------------------------------------
long tc_plane_rows(int B, int T) {
  const long rpad = (long)B * (T + 4);
  return 4 + ((rpad + kTile - 1) / kTile) * kTile;
}
size_t tc_planes_bytes(int B, int T, int c_pad) { return (size_t)(c_pad / 8) * 2 * tc_plane_rows(B, T) * 16; }

int tc_pack_weights(const float* w, int cout, int cin, int taps, int nt_rows, uint8_t** img, cudaStream_t s) {
  const int nchunks = (cin + 63) / 64, n_tiles_n = (cout + nt_rows - 1) / nt_rows;
  const size_t bytes = (size_t)n_tiles_n * nchunks * taps * nt_rows * 256;
  if (!*img) T2_CUDA(cudaMalloc((void**)img, bytes));
  pack_conv_w_kernel<<<n_tiles_n * nchunks * taps, 256, 0, s>>>(w, cout, cin, taps, nt_rows, nchunks, *img);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_rows_to_planes_scaled(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                             __half* planes, const float* in_scale, cudaStream_t s) {
  const long rows = tc_plane_rows(B, T);
  rows_to_planes_kernel<<<dim3((unsigned)((rows + 127) / 128), c_pad / 8), 128, 0, s>>>(x, batch_stride, C, c_pad, len, B, T,
                                                                                      planes, rows, in_scale);
  T2_LAUNCH_CHECK();
  return T2_OK;
}
int tc_rows_to_planes(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                      __half* planes, cudaStream_t s) {
  return tc_rows_to_planes_scaled(x, batch_stride, C, c_pad, len, B, T, planes, nullptr, s);
}

int tc_embed_to_planes(const int64_t* text, const float* emb, int n_symbols, const int32_t* len, int B, int T,
                       __half* planes, cudaStream_t s) {
  const long rows = tc_plane_rows(B, T);
  embed_to_planes_kernel<<<dim3((unsigned)((rows + 127) / 128), kEnc / 8), 128, 0, s>>>(text, emb, n_symbols, len, B, T,
                                                                                       planes, rows);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_fold_bn(const float* cbias, const float* g, const float* b, const float* mean, const float* var, float eps,
               float* scale, float* shift, int C, cudaStream_t s) {
  fold_bn_bias_kernel<<<(C + 127) / 128, 128, 0, s>>>(cbias, g, b, mean, var, eps, scale, shift, C);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_conv(const TcConvArgs& a, cudaStream_t s) {
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const long rows = tc_plane_rows(a.B, a.T);
  // one segment from plane row 0: tile mt reads the padded rows [128 mt - 2, 128 mt + 130)
  p.nchunks = a.cin_pad / 64;
  p.seg[0] = Seg{a.in, rows, 0, p.nchunks}; p.nseg = 1;
  p.wimg = a.wimg; p.taps = a.taps;
  p.n_tiles_m = (int)((rows - 4) / kTile);
  // the grid covers every tile of the plane (rounded up to the cluster size)
  p.B = a.B; p.T = a.T; p.span = a.T + 4; p.lo = 0; p.hi = p.span; p.len = a.row_len;
  p.scale = a.scale; p.bias = a.shift; p.act = a.act; p.out_mode = a.out_mode; p.cout = a.cout;
  p.out = a.out_planes; p.out_rows = rows;
  p.out_f32 = a.out_f32; p.ldo = a.ldo; p.out_seq_rows = a.out_seq_rows > 0 ? a.out_seq_rows : a.T;
  p.residual = a.residual;
  p.res_batch_stride = a.res_batch_stride ? a.res_batch_stride : (long)a.T * a.cout;
  // weights are packed in stages of nt_rows rows; a CTA covers 2 stages' worth of columns when cout allows
  if (a.nt_rows == 128) return launch_gemm<EPI_CONV, 3, 128, 2>(p, (a.cout + 255) / 256, s);
  if (a.nt_rows == 80) return launch_gemm<EPI_CONV, 3, 80, 1>(p, (a.cout + 79) / 80, s);
  return fail(T2_ERR_INVALID, "tc_conv: unsupported n-tile %d", a.nt_rows);
}

}  // namespace t2
