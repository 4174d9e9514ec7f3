// Tensor-core conv1d / GEMM engine (conv_tc.cu): host-side interface.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace t2 {

struct TcConvArgs {
  const __half* in; int cin_pad;          // input planes, channels padded to a multiple of 64
  const uint8_t* wimg; int taps;          // packed weights (tc_pack_weights); 5 = conv k5, 1 = plain GEMM
  int B, T;
  int cout, nt_rows;                      // output channels; columns per CTA (256 / 128 / 80)
  const float* scale; const float* shift; // per output channel: y = acc * scale + shift
  int act;                                // 0 none, 1 relu, 2 tanh
  int out_mode;                           // 0 planes, 1 fp32 rows (B*T, ldo), 2 fp32 (B, cout, T) + residual
  __half* out_planes;
  float* out_f32; long ldo;
  int out_seq_rows;                       // out_mode 1: output row of (b, t) = b * out_seq_rows + t (0 = T)
  const float* residual; long res_batch_stride;
  const int32_t* row_len;                 // (B) or null: out_mode 0 writes zero rows and out_mode 2 zeros at t >= row_len[b]
};

// bytes of the k8 planes of `channels` channels (a multiple of 8) and `rows` rows: a hi and a lo plane of rows x 8 fp16
// per group of 8 channels
inline size_t planes_bytes(int channels, long rows) { return (size_t)(channels / 8) * 2 * rows * 16; }

long tc_plane_rows(int B, int T);
size_t tc_planes_bytes(int B, int T, int c_pad);
// W (cout, cin, taps) -> img, a buffer of tc_weights_bytes(cout, cin, taps, nt_rows)
size_t tc_weights_bytes(int cout, int cin, int taps, int nt_rows);
int tc_pack_weights(const float* w, int cout, int cin, int taps, int nt_rows, uint8_t* img, cudaStream_t s);
int tc_rows_to_planes(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                      __half* planes, cudaStream_t s);
int tc_rows_to_planes_scaled(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                             __half* planes, const float* in_scale /* device scalar or null */, cudaStream_t s);
int tc_embed_to_planes(const int64_t* text, const float* emb, int n_symbols, const int32_t* len /* or null */, int B,
                       int T, __half* planes, cudaStream_t s);
// mel (B, 80, T) fp32 or fp16 -> k8 planes of 16 groups (channels >= 80 zero), `rows` rows: frame f of sequence b at
// plane row guard + b * span + f; frames >= len[b] (len clamped to [0, T]; null: T) and every other row are zero.
// passes 1 writes the hi planes only.
int tc_mel_to_planes(const void* mel, int io_half, int B, int T, const int32_t* len, int guard, int span, __half* planes,
                     long rows, int passes, cudaStream_t s);
int tc_fold_bn(const float* cbias, const float* g, const float* b, const float* mean, const float* var, float eps,
               float* scale, float* shift, int C, cudaStream_t s);
int tc_conv(const TcConvArgs& a, cudaStream_t s);

}  // namespace t2
