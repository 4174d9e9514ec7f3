// Decoder: the control block and the training stash, and the entry points of the stepwise (decoder_stepwise.cu), the
// persistent (decoder_persistent.cu) and the backward (decoder_backward.cu) implementation.
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
  unsigned int q_count; int pad7_[31];     // arrivals of the query CTAs: q of step t written
};

constexpr size_t kDecoderWsAlign = 1024;   // base alignment of a decoder workspace (the persistent slice block)

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

// an attention window or per-row step limits are set (t2b200.h): the persistent kernel's limited instantiation runs
inline bool decoder_has_limits(const T2DecoderArgs* a) { return a->window_front != 0 || a->window_back != 0 || a->max_steps; }

// t2_decoder_workspace_bytes is the larger of the two implementations' layouts
size_t stepwise_ws_bytes(int B, int T);
size_t stepwise_attention_smem(int T);   // the stepwise attention kernel's shared memory (at most 200 KiB: T_enc <= 1282)
size_t persistent_ws_bytes(int B, int T, int cap);
DecoderCtrl* persistent_ws_ctrl(const T2DecoderArgs* a);   // the control block (and phase profile) of a persistent run
int decoder_run_stepwise(T2Model* m, const T2DecoderArgs* a, cudaStream_t s);
// one step of the stepwise decoder (decoder_stepwise.cu), shared by decoder_run_stepwise and t2_decoder_step: the state
// arrays are read and updated in place
struct StepState { float *ah, *ac, *dh, *dc, *aw, *awc, *ctx; };
struct StepIo {
  const float* x2 = nullptr;                   // (B, 256) prenet output
  const float* memory = nullptr; const float* pm = nullptr;
  const int32_t* mem_len = nullptr; const uint8_t* mask = nullptr;
  float score_mask_value = 0.f;
  int B = 0, T = 0;
  int training = 0; const uint8_t* att_keep = nullptr; const uint8_t* dec_keep = nullptr;   // (B, 1024) or Philox
  uint64_t seed = 0; uint32_t site = 0;        // Philox sites site + 2 (attention) and site + 3 (decoder)
  float* gates = nullptr;                      // (B, 4096) scratch
  float* proj = nullptr;                       // (B, 81) out: mel | gate
  float* align_out = nullptr; long align_stride_b = 0;
  const int* skip = nullptr;
};
int decoder_step(T2Model* m, const StepState& st, const StepIo& io, cudaStream_t s);
size_t decoder_step_ws_bytes(int B);
int decoder_step_run(T2Model* m, const T2DecoderStepArgs* a, cudaStream_t s);
int attention_forward(T2Model* m, const T2AttentionArgs* a, cudaStream_t s);
int processed_memory(T2Model* m, const float* memory, int B, int T, float* out, cudaStream_t s);
int decoder_run_persistent(T2Model* m, const T2DecoderArgs* a, cudaStream_t s);
int decoder_backward(T2Model* m, const T2DecoderBwdArgs* a, cudaStream_t s);
size_t decoder_backward_ws_bytes(int B, int T_enc, int T_mel);
size_t prenet_backward_ws_bytes(int M);
int prenet_backward(T2Model* m, const T2PrenetBwdArgs* a, cudaStream_t s);
bool persistent_supported(const T2Model* m, const T2DecoderArgs* a);
// resumable persistent decoder (t2_decoder_stream_*): state = per 64-row slice, status = [steps run, stopped] per slice
size_t persistent_stream_state_bytes(int B, int T_enc);
int persistent_stream_begin(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, cudaStream_t s);
int persistent_stream_run(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, int n, const int32_t* status_host,
                          const int32_t* row_step0, cudaStream_t s);
// continuous batching: rows (ascending) back to the state begin gives them + their processed memory; a chunk's frames of
// the listed rows to the requests' own buffers
int persistent_stream_admit(T2Model* m, const T2DecoderArgs* a, void* state, const int32_t* rows, int n_rows, cudaStream_t s);
int persistent_stream_collect(const T2DecoderArgs* a, const T2CollectRow* rows, int n_rows, cudaStream_t s);
// fp32 rows (n_rows x K, ld) -> split-fp16 activation images of the event engine (event_engine.cuh), one per blockIdx.y;
// grid (K / 64, images) (decoder_persistent.cu)
__global__ void rows_to_image_kernel(const float* __restrict__ src, long ld, int n_rows, int K,
                                     long src_block_stride, uint8_t* __restrict__ dst, long dst_block_stride);

}  // namespace t2
