// Decoder workspace layout shared by the stepwise and the persistent implementation.
#pragma once
#include "model.h"

namespace t2 {

constexpr int kMaxBatch = 1024;

struct DecoderCtrl {
  int all_done;            // every row has fired (INFER) -> remaining work is skipped
  int error;               // device-side watchdog / consistency error code (0 = ok)
  int pad_[2];
  unsigned int bar_count;  // grid barrier of the persistent kernel
  unsigned int bar_gen;
  int pad2_[2];
  int done[kMaxBatch];     // per-row stop latch (SURVEY.md section 8(a) row A9)
  long long prof[3][24];   // cycles per phase of the persistent kernel, sampled on CTAs 0 / 60 / 100
  unsigned int x1_count; int pad3_[31];    // arrivals of the projection CTAs: x1 (and the stop flag) of step t written
  unsigned int x2_count; int pad4_[31];    // arrivals of the prenet-2 CTAs: x2 of step t + 1 written
  unsigned int ah_count[16]; int pad5_[16];   // per 64-column chunk of ah: arrivals of its 8 producer CTAs (8 per step)
  unsigned int dh_count[16]; int pad6_[16];   // the same for dh
};

struct DecoderWs {
  float* pm;               // processed_memory (B, T, 128)          model.py:288
  char* state_begin; size_t state_bytes;   // zero-initialised block (model.py:258-284):
  float *ah, *ac, *dh, *dc;                // (B, 1024) each
  float* ctx;              // (B, 512)
  float *aw, *awc;         // (B, T)
  float *x1, *x2;          // prenet activations (B, 256)
  float* gates;            // (B, 4096)
  float* proj;             // (B, 81)
  DecoderCtrl* ctrl;
  uint8_t* images;         // persistent kernel: activation images and q (decoder_persistent.cu)
  uint8_t* teacher_img;    // persistent kernel, teacher forcing: the x2 images of every step
};
constexpr size_t kDecoderWsAlign = 1024;   // largest alignment of a decoder workspace region (teacher_img)

// Training stash written by the persistent kernel in teacher-forced mode and read by the backward pass
// (decoder_backward.cu).  All fp32, step-major.  h = the hidden state that recurs (after dropout).
struct DecoderStash {
  float* ga = nullptr; float* gd = nullptr;                   // (T, B, 4096) gate activations i | f | g | o
  float* ca = nullptr; float* ha = nullptr;                   // (T + 1, B, 1024), slot 0 = initial zeros
  float* cd = nullptr; float* hd = nullptr;
  float* ctx = nullptr;                                       // (T + 1, B, 512), slot 0 = zeros
};
inline void decoder_stash_layout(Carve& c, int B, int T, DecoderStash* s) {
  s->ga = c.take<float>((size_t)T * B * 4096); s->gd = c.take<float>((size_t)T * B * 4096);
  s->ca = c.take<float>((size_t)(T + 1) * B * 1024); s->ha = c.take<float>((size_t)(T + 1) * B * 1024);
  s->cd = c.take<float>((size_t)(T + 1) * B * 1024); s->hd = c.take<float>((size_t)(T + 1) * B * 1024);
  s->ctx = c.take<float>((size_t)(T + 1) * B * 512);
}
inline size_t decoder_stash_bytes(int B, int T) { Carve c(nullptr); DecoderStash s; decoder_stash_layout(c, B, T, &s); return c.bytes(); }

size_t decoder_ws_bytes(int B, int T, int cap);
void persistent_ws_layout(Carve& c, int cap, DecoderWs* w);
int decoder_ws_carve(const T2DecoderArgs* a, DecoderWs* w);
int decoder_run_stepwise(T2Model* m, const T2DecoderArgs* a, cudaStream_t s);
int decoder_run_persistent(T2Model* m, const T2DecoderArgs* a, cudaStream_t s);
int decoder_backward(T2Model* m, const T2DecoderBwdArgs* a, cudaStream_t s);
size_t decoder_backward_ws_bytes(int B, int T_enc, int T_mel);
size_t prenet_backward_ws_bytes(int M);
int prenet_backward(T2Model* m, const T2PrenetBwdArgs* a, cudaStream_t s);
bool persistent_supported(const T2Model* m, const T2DecoderArgs* a);
// resumable persistent decoder (t2_decoder_stream_*): state = per 64-row slice, status = [steps run, stopped] per slice
size_t persistent_stream_state_bytes(int B, int T_enc);
int persistent_stream_begin(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, cudaStream_t s);
int persistent_stream_run(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, int n,
                          const int32_t* status_host, cudaStream_t s);
// continuous batching: rows (ascending) back to the state begin gives them + their processed memory; a chunk's frames of
// the listed rows to the requests' own buffers
int persistent_stream_admit(T2Model* m, const T2DecoderArgs* a, void* state, const int32_t* rows, int n_rows, cudaStream_t s);
int persistent_stream_collect(const T2DecoderArgs* a, const T2CollectRow* rows, int n_rows, cudaStream_t s);

// tensor-core skinny GEMMs of the decoder backward (decoder_persistent.cu): which = 0 decoder LSTM (2560 columns),
// 1 attention LSTM (1792 columns); K = 4096 gate rows in kBwdGemmSplit partial sums
constexpr int kBwdGemmSplit = 4;
constexpr int kBwdImgBytes = 64 * 16384;     // activation image of one (64 x 4096) operand
int bwd_gemm_prepare(T2Model* m, cudaStream_t s);
int bwd_gemm_run(T2Model* m, int which, const uint8_t* x_img, const float* inv_scale, float* P, int ldp, DecoderCtrl* ctrl,
                 cudaStream_t s);

}  // namespace t2
