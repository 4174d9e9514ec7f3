// T2Model: configuration, caller's fp32 weight pointers and the packed device-side copies.
#pragma once
#include "common.cuh"

struct T2Model {
  T2Config cfg;
  int device = 0;
  int sm_count = 0;
  const float* w[t2::W_COUNT];   // caller-owned fp32 state_dict tensors (device)

  // ---- packed fp32 copies (owned) ----
  float* enc_conv_w[3] = {};     // (512, 5, 512)  [co][tap][ci]
  float* post_conv_w[5] = {};    // (co, 5, ci)
  float* enc_lstm_wih = nullptr; // (2048, 512): forward rows then reverse rows
  float* enc_lstm_b = nullptr;   // (2048): b_ih + b_hh, forward then reverse
  float* arnn_b = nullptr;       // (4096) b_ih + b_hh
  float* drnn_b = nullptr;       // (4096)
  float* projgate_w = nullptr;   // (81, 1536): linear_projection rows then the gate row
  float* projgate_b = nullptr;   // (81)
  float* zeros = nullptr;        // >= 4096 zeros (go frame etc.)

  // ---- tensor-core conv / GEMM weight images (conv_tc.cu) ----
  uint8_t* tc_enc_conv[3] = {};  // (512, 512, 5)  n-tile 256
  uint8_t* tc_enc_wih = nullptr; // (2048, 512)    n-tile 256, taps = 1
  uint8_t* tc_post_conv[5] = {}; // n-tile 256 (layers 0-3), 80 (layer 4)
  // training: input-gradient convolutions = the same engine with flipped / transposed weights (re-packed per backward)
  uint8_t* tc_dgrad_enc[3] = {}; uint8_t* tc_dgrad_post[5] = {};
  float* dgrad_tmp = nullptr;    // (512, 512, 5) fp32 scratch for the flipped weights

  // ---- packed operands of the persistent decoder kernel (owned; see decoder_persistent.cu) ----
  void* pk = nullptr;            // opaque PersistentPack*
  void* gemm_ws = nullptr; size_t gemm_ws_bytes = 0;   // scratch of gemm_tc.cu (operand scales, split-K partial tiles)
};

namespace t2 {
int pack_model(T2Model* m, cudaStream_t s);          // (re)builds every packed copy
int persistent_pack_create(T2Model* m, cudaStream_t s);
void persistent_pack_destroy(T2Model* m);
}  // namespace t2
