// C ABI of libt2b200.so (include/t2b200.h): argument checking, weight packing, dispatch.
#include <stdarg.h>
#include <string.h>

#include <vector>

#include "conv_tc.h"
#include "decoder.h"
#include "gemm_tc.h"
#include "gemm_f32.cuh"
#include "train_layers.h"
#include "waveglow.h"
#include "denoiser.h"

namespace t2 {

std::string& last_error() {
  static thread_local std::string e;
  return e;
}
long long g_launch_count = 0;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}

int encoder_forward(T2Model* m, const T2EncoderArgs* a, cudaStream_t s, bool per_row);
size_t encoder_ws_bytes(int B, int T);
int postnet_forward(T2Model* m, const T2PostnetArgs* a, cudaStream_t s, bool per_row);
size_t postnet_ws_bytes(int B, int T);
int selftest_umma(const float* A, const float* W, int N, int K, int passes, float* C, cudaStream_t s);
int selftest_event(const float* A, const float* W, const int* cons, int ncons, int K, float* C, cudaStream_t s);
int mma_rate(int M, int N, int reps, int alternate_d, long long* out_host, cudaStream_t s);
int mma_group(int M, int N, int group, int reps, long long* out_host, cudaStream_t s);

// ---- weight packing -----------------------------------------------------------------------------
// conv weight (co, ci, k) -> (co, k, ci) so a conv is a GEMM over K = taps x Cin on channels-last rows
__global__ void permute_conv_kernel(const float* __restrict__ w, float* __restrict__ out, int co, int ci, int k) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)co * ci * k) return;
  const int kk = (int)(i % k); const long r = i / k; const int c = (int)(r % ci); const int o = (int)(r / ci);
  out[((long)o * k + kk) * ci + c] = w[i];
}
__global__ void add2_kernel(const float* a, const float* b, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

template <typename T>
static int dmalloc(T** p, size_t n) {
  if (*p) return T2_OK;
  T2_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
  return T2_OK;
}

int pack_model(T2Model* m, cudaStream_t s) {
  for (int i = 0; i < 3; ++i) {
    T2_TRY(dmalloc(&m->enc_conv_w[i], (size_t)kEnc * kEnc * kConvK));
    const long n = (long)kEnc * kEnc * kConvK;
    permute_conv_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(m->w[W_ENC_CONV0 + 7 * i], m->enc_conv_w[i], kEnc, kEnc, kConvK);
    T2_LAUNCH_CHECK();
  }
  for (int i = 0; i < 5; ++i) {
    const int ci = i == 0 ? kMel : kPost, co = i == 4 ? kMel : kPost;
    T2_TRY(dmalloc(&m->post_conv_w[i], (size_t)co * ci * kConvK));
    const long n = (long)co * ci * kConvK;
    permute_conv_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(m->w[W_POST_CONV0 + 7 * i], m->post_conv_w[i], co, ci, kConvK);
    T2_LAUNCH_CHECK();
  }
  T2_TRY(dmalloc(&m->enc_lstm_wih, (size_t)8 * kEncH * kEnc));
  T2_TRY(dmalloc(&m->enc_lstm_b, (size_t)8 * kEncH));
  for (int d = 0; d < 2; ++d) {
    T2_CUDA(cudaMemcpyAsync(m->enc_lstm_wih + (size_t)d * 4 * kEncH * kEnc, m->w[W_ENC_LSTM + 4 * d],
                            (size_t)4 * kEncH * kEnc * 4, cudaMemcpyDeviceToDevice, s));
    add2_kernel<<<(4 * kEncH + 255) / 256, 256, 0, s>>>(m->w[W_ENC_LSTM + 4 * d + 2], m->w[W_ENC_LSTM + 4 * d + 3],
                                                        m->enc_lstm_b + d * 4 * kEncH, 4 * kEncH);
    T2_LAUNCH_CHECK();
  }
  T2_TRY(dmalloc(&m->arnn_b, (size_t)4 * kARnn));
  T2_TRY(dmalloc(&m->drnn_b, (size_t)4 * kDRnn));
  add2_kernel<<<(4 * kARnn + 255) / 256, 256, 0, s>>>(m->w[W_ARNN_BIH], m->w[W_ARNN_BHH], m->arnn_b, 4 * kARnn);
  T2_LAUNCH_CHECK();
  add2_kernel<<<(4 * kDRnn + 255) / 256, 256, 0, s>>>(m->w[W_DRNN_BIH], m->w[W_DRNN_BHH], m->drnn_b, 4 * kDRnn);
  T2_LAUNCH_CHECK();
  const int kdc = kDRnn + kEnc;
  T2_TRY(dmalloc(&m->projgate_w, (size_t)(kMel + 1) * kdc));
  T2_TRY(dmalloc(&m->projgate_b, (size_t)(kMel + 1)));
  T2_CUDA(cudaMemcpyAsync(m->projgate_w, m->w[W_PROJ_W], (size_t)kMel * kdc * 4, cudaMemcpyDeviceToDevice, s));
  T2_CUDA(cudaMemcpyAsync(m->projgate_w + (size_t)kMel * kdc, m->w[W_GATE_W], (size_t)kdc * 4, cudaMemcpyDeviceToDevice, s));
  T2_CUDA(cudaMemcpyAsync(m->projgate_b, m->w[W_PROJ_B], kMel * 4, cudaMemcpyDeviceToDevice, s));
  T2_CUDA(cudaMemcpyAsync(m->projgate_b + kMel, m->w[W_GATE_B], 4, cudaMemcpyDeviceToDevice, s));
  if (!m->zeros) {
    T2_TRY(dmalloc(&m->zeros, (size_t)8192));
    T2_CUDA(cudaMemsetAsync(m->zeros, 0, 8192 * 4, s));
  }
  // tensor-core conv / GEMM weight images
  for (int i = 0; i < 3; ++i) T2_TRY(tc_pack_weights(m->w[W_ENC_CONV0 + 7 * i], kEnc, kEnc, kConvK, 128, &m->tc_enc_conv[i], s));
  T2_TRY(tc_pack_weights(m->enc_lstm_wih, 8 * kEncH, kEnc, 1, 128, &m->tc_enc_wih, s));
  for (int i = 0; i < 5; ++i) {
    const int ci = i == 0 ? kMel : kPost, co = i == 4 ? kMel : kPost;
    T2_TRY(tc_pack_weights(m->w[W_POST_CONV0 + 7 * i], co, ci, kConvK, i == 4 ? 80 : 128, &m->tc_post_conv[i], s));
  }
  T2_TRY(persistent_pack_create(m, s));
  return T2_OK;
}

// ---- decoder workspace --------------------------------------------------------------------------
static void decoder_ws_layout(Carve& c, int B, int T, int cap, DecoderWs* w) {
  w->pm = c.take<float>((size_t)B * T * kAtt);
  // the zero-initialised states: packed floats, one block that one memset clears
  w->state_begin = c.take<char>(0);
  const size_t state0 = c.off;
  w->ah = c.take<float>((size_t)B * kARnn, alignof(float)); w->ac = c.take<float>((size_t)B * kARnn, alignof(float));
  w->dh = c.take<float>((size_t)B * kDRnn, alignof(float)); w->dc = c.take<float>((size_t)B * kDRnn, alignof(float));
  w->ctx = c.take<float>((size_t)B * kEnc, alignof(float));
  w->aw = c.take<float>((size_t)B * T, alignof(float)); w->awc = c.take<float>((size_t)B * T, alignof(float));
  w->state_bytes = c.off - state0;
  w->x1 = c.take<float>((size_t)B * kPre); w->x2 = c.take<float>((size_t)B * kPre);
  w->gates = c.take<float>((size_t)B * 4 * kARnn);
  w->proj = c.take<float>((size_t)B * (kMel + 1));
  w->ctrl = c.take<DecoderCtrl>(1);
  persistent_ws_layout(c, cap, w);
}

size_t decoder_ws_bytes(int B, int T, int cap) {
  Carve c(nullptr, kDecoderWsAlign);
  DecoderWs w;
  decoder_ws_layout(c, B, T, cap, &w);
  return c.bytes();
}

int decoder_ws_carve(const T2DecoderArgs* a, DecoderWs* w) {
  if (a->ws_bytes < decoder_ws_bytes(a->B, a->T_enc, a->n_steps_cap)) return fail(T2_ERR_WORKSPACE, "decoder workspace too small");
  Carve c(a->ws, kDecoderWsAlign);
  decoder_ws_layout(c, a->B, a->T_enc, a->n_steps_cap, w);
  return T2_OK;
}

static int check_decoder_args(const T2Model* m, const T2DecoderArgs* a) {
  if (!m || !a) return fail(T2_ERR_INVALID, "null model / args");
  if (a->B <= 0 || a->B > kMaxBatch) return fail(T2_ERR_INVALID, "decoder: B=%d outside [1, %d]", a->B, kMaxBatch);
  if (a->T_enc <= 0) return fail(T2_ERR_INVALID, "decoder: empty encoder memory (T_enc=%d)", a->T_enc);
  if (a->n_steps_cap <= 0) return fail(T2_ERR_INVALID, "decoder: n_steps_cap=%d", a->n_steps_cap);
  if (!a->memory || !a->mel || !a->gate || !a->align || !a->mel_lengths || !a->n_steps || !a->ws)
    return fail(T2_ERR_INVALID, "decoder: null tensor pointer");
  if (a->mode == T2_MODE_TEACHER && !a->teacher_prenet) return fail(T2_ERR_INVALID, "decoder: teacher mode needs teacher_prenet");
  if (a->mode != T2_MODE_TEACHER && a->mode != T2_MODE_INFER) return fail(T2_ERR_INVALID, "decoder: bad mode %d", a->mode);
  return T2_OK;
}

}  // namespace t2

using namespace t2;

extern "C" {

int t2_abi_version(void) { return T2_ABI_VERSION; }
const char* t2_last_error(void) { return last_error().c_str(); }
int64_t t2_kernel_launch_count(void) { return g_launch_count; }

int t2_device_info(int32_t out[5]) {
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  out[0] = p.multiProcessorCount; out[1] = p.major; out[2] = p.minor;
  out[3] = (int32_t)(p.l2CacheSize); out[4] = (int32_t)p.sharedMemPerBlockOptin;
  return T2_OK;
}

static int check_cfg(const T2Config* c) {
  const bool ok = c->n_mel_channels == kMel && c->symbols_embedding_dim == kEnc && c->encoder_kernel_size == kConvK &&
                  c->encoder_n_convolutions == 3 && c->encoder_embedding_dim == kEnc && c->attention_rnn_dim == kARnn &&
                  c->decoder_rnn_dim == kDRnn && c->prenet_dim == kPre && c->attention_dim == kAtt &&
                  c->attention_location_n_filters == kLocF && c->attention_location_kernel_size == kLocK &&
                  c->postnet_embedding_dim == kPost && c->postnet_kernel_size == kConvK && c->postnet_n_convolutions == 5 &&
                  c->n_symbols > 0;
  if (!ok) return fail(T2_ERR_UNSUPPORTED, "hyper-parameters differ from the reference defaults the sm_90a kernels are built for");
  return T2_OK;
}

static int set_weights(T2Model* m, const void* const* weights, int32_t n) {
  if (n != T2_NUM_WEIGHTS) return fail(T2_ERR_INVALID, "expected %d weight pointers, got %d", T2_NUM_WEIGHTS, n);
  for (int i = 0; i < n; ++i) {
    const bool nbt = (i >= W_ENC_CONV0 && i < W_ENC_LSTM && (i - W_ENC_CONV0) % 7 == 6) ||
                     (i >= W_POST_CONV0 && (i - W_POST_CONV0) % 7 == 6);
    if (!nbt && weights[i] == nullptr) return fail(T2_ERR_INVALID, "weight %d is null", i);
    m->w[i] = (const float*)weights[i];
  }
  return T2_OK;
}

int t2_model_create(T2Model** out, const T2Config* cfg, const void* const* weights, int32_t n_weights, void* stream) {
  if (!out || !cfg || !weights) return fail(T2_ERR_INVALID, "null argument");
  T2_TRY(check_cfg(cfg));
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) return fail(T2_ERR_UNSUPPORTED, "libt2b200 is built for sm_90a only (device is sm_%d%d)", p.major, p.minor);
  T2Model* m = new T2Model();
  m->cfg = *cfg; m->device = dev; m->sm_count = p.multiProcessorCount;
  int r = set_weights(m, weights, n_weights);
  if (r == T2_OK) r = pack_model(m, (cudaStream_t)stream);
  if (r != T2_OK) { t2_model_destroy(m); return r; }
  *out = m;
  return T2_OK;
}

int t2_model_refresh(T2Model* m, const void* const* weights, int32_t n_weights, void* stream) {
  if (!m) return fail(T2_ERR_INVALID, "null model");
  T2_TRY(set_weights(m, weights, n_weights));
  return pack_model(m, (cudaStream_t)stream);
}

int t2_model_destroy(T2Model* m) {
  if (!m) return T2_OK;
  for (int i = 0; i < 3; ++i) cudaFree(m->enc_conv_w[i]);
  for (int i = 0; i < 5; ++i) cudaFree(m->post_conv_w[i]);
  cudaFree(m->enc_lstm_wih); cudaFree(m->enc_lstm_b); cudaFree(m->arnn_b); cudaFree(m->drnn_b);
  cudaFree(m->projgate_w); cudaFree(m->projgate_b); cudaFree(m->zeros); cudaFree(m->dgrad_tmp);
  for (int i = 0; i < 3; ++i) cudaFree(m->tc_dgrad_enc[i]);
  for (int i = 0; i < 5; ++i) cudaFree(m->tc_dgrad_post[i]);
  for (int i = 0; i < 3; ++i) cudaFree(m->tc_enc_conv[i]);
  for (int i = 0; i < 5; ++i) cudaFree(m->tc_post_conv[i]);
  cudaFree(m->tc_enc_wih);
  persistent_pack_destroy(m);
  gemm_tc_destroy(m);
  delete m;
  return T2_OK;
}

size_t t2_encoder_workspace_bytes(const T2Model*, int32_t B, int32_t T) { return encoder_ws_bytes(B, T); }
int t2_encoder_forward(T2Model* m, const T2EncoderArgs* a, void* stream) {
  if (!m || !a || (!a->text && !a->embedded) || !a->memory || !a->ws) return fail(T2_ERR_INVALID, "encoder: null argument");
  return encoder_forward(m, a, (cudaStream_t)stream, false);
}

int t2_encoder_infer(T2Model* m, const T2EncoderArgs* a, void* stream) {
  if (!m || !a || (!a->text && !a->embedded) || !a->memory || !a->ws) return fail(T2_ERR_INVALID, "encoder infer: null argument");
  if (a->training || a->stash) return fail(T2_ERR_INVALID, "encoder infer: evaluation only (training = 0, no stash)");
  return encoder_forward(m, a, (cudaStream_t)stream, true);
}

size_t t2_encoder_stash_bytes(const T2Model*, int32_t B, int32_t T) { return encoder_stash_bytes(B, T); }
size_t t2_encoder_backward_workspace_bytes(const T2Model*, int32_t B, int32_t T) { return encoder_backward_ws_bytes(B, T); }
int t2_encoder_backward(T2Model* m, const T2EncoderBwdArgs* a, void* stream) {
  if (!m || !a || (!a->text && !a->embedded) || !a->stash || !a->d_memory || !a->grads || !a->ws)
    return fail(T2_ERR_INVALID, "encoder backward: null argument");
  return encoder_backward(m, a, (cudaStream_t)stream);
}
size_t t2_postnet_stash_bytes(const T2Model*, int32_t B, int32_t T) { return postnet_stash_bytes(B, T); }
size_t t2_postnet_backward_workspace_bytes(const T2Model*, int32_t B, int32_t T) { return postnet_backward_ws_bytes(B, T); }
int t2_postnet_backward(T2Model* m, const T2PostnetBwdArgs* a, void* stream) {
  if (!m || !a || !a->stash || !a->d_mel_post || !a->grads || !a->ws) return fail(T2_ERR_INVALID, "postnet backward: null argument");
  return postnet_backward(m, a, (cudaStream_t)stream);
}

size_t t2_decoder_workspace_bytes(const T2Model*, int32_t B, int32_t T_enc, int32_t cap) { return decoder_ws_bytes(B, T_enc, cap); }
int t2_decoder_run(T2Model* m, const T2DecoderArgs* a, void* stream) {
  T2_TRY(check_decoder_args(m, a));
  int impl = a->impl;
  if (impl == T2_IMPL_AUTO) impl = persistent_supported(m, a) ? T2_IMPL_PERSISTENT : T2_IMPL_STEPWISE;
  if (impl == T2_IMPL_PERSISTENT) {
    if (!persistent_supported(m, a))
      return fail(T2_ERR_UNSUPPORTED, "persistent decoder does not support T_enc=%d on this device (at most 2274, and >= 128 SMs)",
                  a->T_enc);
    return decoder_run_persistent(m, a, (cudaStream_t)stream);
  }
  // only the persistent kernel writes the training stash: a backward pass over a stash the stepwise path left
  // untouched would silently produce garbage gradients
  if (a->stash)
    return fail(T2_ERR_UNSUPPORTED, "decoder: the training stash needs the persistent implementation (%s)",
                a->impl == T2_IMPL_STEPWISE ? "impl = STEPWISE was requested"
                                            : "this shape / device does not fit it: T_enc too large for shared memory or < 128 SMs");
  return decoder_run_stepwise(m, a, (cudaStream_t)stream);
}

size_t t2_decoder_stream_state_bytes(const T2Model*, int32_t B, int32_t T_enc) {
  return B > 0 && T_enc > 0 ? persistent_stream_state_bytes(B, T_enc) : 0;
}

static int check_stream_args(const T2Model* m, const T2DecoderStreamArgs* s) {
  if (!m || !s) return fail(T2_ERR_INVALID, "decoder stream: null model / args");
  const T2DecoderArgs* a = &s->dec;
  if (a->B <= 0 || a->B > kMaxBatch) return fail(T2_ERR_INVALID, "decoder stream: B=%d outside [1, %d]", a->B, kMaxBatch);
  if (a->T_enc <= 0) return fail(T2_ERR_INVALID, "decoder stream: empty encoder memory (T_enc=%d)", a->T_enc);
  if (a->n_steps_cap <= 0) return fail(T2_ERR_INVALID, "decoder stream: n_steps_cap=%d", a->n_steps_cap);
  if (!a->memory || !a->mel || !a->gate || !a->align || !a->mel_lengths || !a->n_steps || !s->state || !s->status)
    return fail(T2_ERR_INVALID, "decoder stream: null tensor pointer");
  if (a->mode != T2_MODE_INFER) return fail(T2_ERR_INVALID, "decoder stream: mode must be INFER (got %d)", a->mode);
  if (a->impl == T2_IMPL_STEPWISE)
    return fail(T2_ERR_UNSUPPORTED, "decoder stream: needs the persistent decoder, which resumes from saved state "
                                    "(impl = STEPWISE was requested)");
  if (a->impl != T2_IMPL_AUTO && a->impl != T2_IMPL_PERSISTENT) return fail(T2_ERR_INVALID, "decoder stream: bad impl %d", a->impl);
  if (!persistent_supported(m, a))
    return fail(T2_ERR_UNSUPPORTED, "decoder stream: the persistent decoder does not support T_enc=%d on this device "
                                    "(at most 2274, and >= 128 SMs)", a->T_enc);
  if (s->state_bytes < persistent_stream_state_bytes(a->B, a->T_enc)) return fail(T2_ERR_WORKSPACE, "decoder stream state too small");
  return T2_OK;
}

int t2_decoder_stream_begin(T2Model* m, const T2DecoderStreamArgs* a, void* stream) {
  T2_TRY(check_stream_args(m, a));
  return persistent_stream_begin(m, &a->dec, a->state, a->status, (cudaStream_t)stream);
}

int t2_decoder_stream_run(T2Model* m, const T2DecoderStreamArgs* a, int32_t n_steps, const int32_t* status_host, void* stream) {
  T2_TRY(check_stream_args(m, a));
  if (n_steps < 1) return fail(T2_ERR_INVALID, "decoder stream: n_steps=%d (at least 1 step per run)", n_steps);
  return persistent_stream_run(m, &a->dec, a->state, a->status, n_steps, status_host, (cudaStream_t)stream);
}

int t2_decoder_stream_admit(T2Model* m, const T2DecoderStreamArgs* a, const int32_t* rows, int32_t n_rows, void* stream) {
  T2_TRY(check_stream_args(m, a));
  if (n_rows < 1 || n_rows > a->dec.B || !rows) return fail(T2_ERR_INVALID, "decoder stream admit: n_rows=%d outside [1, B=%d]", n_rows, a->dec.B);
  if (!a->dec.memory_lengths) return fail(T2_ERR_INVALID, "decoder stream admit: the stream has no memory_lengths");
  for (int i = 0; i < n_rows; ++i)
    if (rows[i] < 0 || rows[i] >= a->dec.B || (i > 0 && rows[i] <= rows[i - 1]))
      return fail(T2_ERR_INVALID, "decoder stream admit: rows must be ascending and inside [0, B=%d) (rows[%d]=%d)", a->dec.B, i, rows[i]);
  return persistent_stream_admit(m, &a->dec, a->state, rows, n_rows, (cudaStream_t)stream);
}

int t2_decoder_stream_collect(T2Model* m, const T2DecoderStreamArgs* a, const T2CollectRow* rows, int32_t n_rows, void* stream) {
  T2_TRY(check_stream_args(m, a));
  if (n_rows < 1 || n_rows > a->dec.B || !rows) return fail(T2_ERR_INVALID, "decoder stream collect: n_rows=%d outside [1, B=%d]", n_rows, a->dec.B);
  for (int i = 0; i < n_rows; ++i) {
    const T2CollectRow& r = rows[i];
    if (r.row < 0 || r.row >= a->dec.B || r.n_frames < 0 || r.n_frames > a->dec.n_steps_cap || r.T_text < 1 || r.T_text > a->dec.T_enc)
      return fail(T2_ERR_INVALID, "decoder stream collect: entry %d (row %d, %d frames, T_text %d) outside B=%d, n_steps_cap=%d, T_enc=%d",
                  i, r.row, r.n_frames, r.T_text, a->dec.B, a->dec.n_steps_cap, a->dec.T_enc);
    if (!r.mel || !r.gate || !r.align) return fail(T2_ERR_INVALID, "decoder stream collect: entry %d has a null destination", i);
  }
  return persistent_stream_collect(&a->dec, rows, n_rows, (cudaStream_t)stream);
}

size_t t2_decoder_stash_bytes(const T2Model*, int32_t B, int32_t, int32_t T_mel) { return decoder_stash_bytes(B, T_mel); }
size_t t2_decoder_backward_workspace_bytes(const T2Model*, int32_t B, int32_t T_enc, int32_t T_mel) {
  return decoder_backward_ws_bytes(B, T_enc, T_mel);
}
int t2_decoder_backward(T2Model* m, const T2DecoderBwdArgs* a, void* stream) {
  if (!m || !a || !a->memory || !a->teacher_prenet || !a->align || !a->stash || !a->d_mel || !a->d_gate || !a->d_prenet ||
      !a->grads || !a->ws)
    return fail(T2_ERR_INVALID, "decoder backward: null argument");
  return decoder_backward(m, a, (cudaStream_t)stream);
}
size_t t2_prenet_backward_workspace_bytes(const T2Model*, int32_t M) { return prenet_backward_ws_bytes(M); }
int t2_prenet_backward(T2Model* m, const T2PrenetBwdArgs* a, void* stream) {
  if (!m || !a || !a->frames || !a->d_out || !a->grads || !a->ws || a->M <= 0) return fail(T2_ERR_INVALID, "prenet backward: bad argument");
  return prenet_backward(m, a, (cudaStream_t)stream);
}

int t2_prenet_forward(T2Model* m, const float* frames, int32_t M, const uint8_t* keep, uint64_t seed, float* out,
                      void* ws, size_t ws_bytes, void* stream) {
  if (!m || !frames || !out || M <= 0) return fail(T2_ERR_INVALID, "prenet: bad argument");
  if (ws_bytes < (size_t)M * kPre * 4) return fail(T2_ERR_WORKSPACE, "prenet workspace too small");
  float* x1 = (float*)ws;
  GemmArgs g;                                                     // model.py:97-100
  g.seg[0] = {frames, kMel, m->w[W_PRENET0], kMel, kMel};
  g.M = M; g.N = kPre; g.C = x1; g.ldc = kPre; g.act = ACT_RELU; g.p_drop = 0.5f;
  if (keep) { g.keep = keep; g.ldkeep = kPre; } else { g.philox = 1; g.seed = seed; g.site = 0xA0; }
  T2_TRY(gemm_f32(g, (cudaStream_t)stream));
  GemmArgs h;
  h.seg[0] = {x1, kPre, m->w[W_PRENET1], kPre, kPre};
  h.M = M; h.N = kPre; h.C = out; h.ldc = kPre; h.act = ACT_RELU; h.p_drop = 0.5f;
  if (keep) { h.keep = keep + (size_t)M * kPre; h.ldkeep = kPre; } else { h.philox = 1; h.seed = seed; h.site = 0xA1; }
  return gemm_f32(h, (cudaStream_t)stream);
}

size_t t2_postnet_workspace_bytes(const T2Model*, int32_t B, int32_t T) { return postnet_ws_bytes(B, T); }
int t2_postnet_forward(T2Model* m, const T2PostnetArgs* a, void* stream) {
  if (!m || !a || !a->mel || !a->mel_post || !a->ws) return fail(T2_ERR_INVALID, "postnet: null argument");
  return postnet_forward(m, a, (cudaStream_t)stream, false);
}

int t2_postnet_infer(T2Model* m, const T2PostnetArgs* a, void* stream) {
  if (!m || !a || !a->mel || !a->mel_post || !a->ws) return fail(T2_ERR_INVALID, "postnet infer: null argument");
  if (a->training || a->stash) return fail(T2_ERR_INVALID, "postnet infer: evaluation only (training = 0, no stash)");
  return postnet_forward(m, a, (cudaStream_t)stream, true);
}

// ---- end to end with host buffers ------------------------------------------------------------------
struct InferWs {
  int64_t* text; float *memory, *mel, *gate, *align, *post; int32_t *lens, *nsteps;
  char* sub; size_t sub_bytes;   // the workspace of the encoder, the decoder and the postnet in turn
  int32_t* in_lens;              // t2_infer_host_lengths: the input lengths (B)
};
static void infer_layout(Carve& c, int B, int Tt, int S, InferWs* w, bool with_lengths = false) {
  w->text = c.take<int64_t>((size_t)B * Tt);
  w->memory = c.take<float>((size_t)B * Tt * kEnc);
  w->mel = c.take<float>((size_t)B * S * kMel);
  w->gate = c.take<float>((size_t)B * S);
  w->align = c.take<float>((size_t)B * S * Tt);
  w->post = c.take<float>((size_t)B * S * kMel);
  w->lens = c.take<int32_t>(B);
  w->nsteps = c.take<int32_t>(1);
  size_t sb = encoder_ws_bytes(B, Tt);
  if (decoder_ws_bytes(B, Tt, S) > sb) sb = decoder_ws_bytes(B, Tt, S);
  if (postnet_ws_bytes(B, S) > sb) sb = postnet_ws_bytes(B, S);
  w->sub = c.take<char>(sb); w->sub_bytes = sb;
  w->in_lens = with_lengths ? c.take<int32_t>(B) : nullptr;
}

size_t t2_infer_workspace_bytes(const T2Model*, int32_t B, int32_t T_text, int32_t max_steps) {
  Carve c(nullptr);
  InferWs w;
  infer_layout(c, B, T_text, max_steps, &w);
  return c.bytes();
}

size_t t2_infer_lengths_workspace_bytes(const T2Model*, int32_t B, int32_t T_text, int32_t max_steps) {
  Carve c(nullptr);
  InferWs w;
  infer_layout(c, B, T_text, max_steps, &w, true);
  return c.bytes();
}

// Tacotron2.inference end to end; in_lens_host (B) or null: each row b is its first in_lens_host[b] symbols alone
static int infer_host(T2Model* m, const int64_t* text_host, const int64_t* in_lens_host, int32_t B, int32_t T_text,
                      int32_t max_steps, float gate_threshold, uint64_t seed, int32_t impl, float* mel_post_host,
                      int32_t* mel_lengths_host, int32_t* n_steps_host, void* ws, size_t ws_bytes, cudaStream_t s) {
  if (!m || !text_host || !mel_post_host || !mel_lengths_host || !n_steps_host || !ws)
    return fail(T2_ERR_INVALID, "infer_host: null argument");
  const bool with_lengths = in_lens_host != nullptr;
  const size_t need = with_lengths ? t2_infer_lengths_workspace_bytes(m, B, T_text, max_steps)
                                   : t2_infer_workspace_bytes(m, B, T_text, max_steps);
  if (ws_bytes < need) return fail(T2_ERR_WORKSPACE, "infer workspace too small");
  std::vector<int32_t> lens32;
  bool ragged = false;             // some text shorter than T_text: each row's postnet is its own B = 1 postnet
  if (with_lengths) {              // checked here, before anything is enqueued
    lens32.resize(B > 0 ? B : 0);
    for (int b = 0; b < B; ++b) {
      if (in_lens_host[b] < 1 || in_lens_host[b] > T_text)
        return fail(T2_ERR_INVALID, "infer_host: input_lengths[%d] = %lld outside [1, %d]", b, (long long)in_lens_host[b], T_text);
      lens32[b] = (int32_t)in_lens_host[b];
      ragged |= lens32[b] < T_text;
    }
  }
  Carve c(ws);
  InferWs w;
  infer_layout(c, B, T_text, max_steps, &w, with_lengths);
  T2_CUDA(cudaMemcpyAsync(w.text, text_host, (size_t)B * T_text * 8, cudaMemcpyHostToDevice, s));
  // pageable source: the call returns once lens32 has been staged, so the vector may go out of scope
  if (with_lengths) T2_CUDA(cudaMemcpyAsync(w.in_lens, lens32.data(), (size_t)B * 4, cudaMemcpyHostToDevice, s));
  T2EncoderArgs ea; memset(&ea, 0, sizeof(ea));
  ea.text = w.text; ea.lengths = w.in_lens; ea.B = B; ea.T = T_text; ea.memory = w.memory; ea.ws = w.sub; ea.ws_bytes = w.sub_bytes;
  T2_TRY(encoder_forward(m, &ea, s, true));
  T2DecoderArgs da; memset(&da, 0, sizeof(da));
  da.mode = T2_MODE_INFER; da.impl = impl; da.memory = w.memory; da.memory_lengths = w.in_lens;
  da.B = B; da.T_enc = T_text; da.n_steps_cap = max_steps;
  da.seed = seed; da.gate_threshold = gate_threshold; da.score_mask_value = -INFINITY;
  da.mel = w.mel; da.gate = w.gate; da.align = w.align; da.mel_lengths = w.lens; da.n_steps = w.nsteps; da.ws = w.sub; da.ws_bytes = w.sub_bytes;
  T2_TRY(t2_decoder_run(m, &da, s));
  // the postnet runs over the n decoded frames, as Tacotron2.inference does: its convolutions zero-pad every layer at
  // frame n, and a longer window would feed the last rows' final frames the activations of zero input instead
  T2_CUDA(cudaMemcpyAsync(n_steps_host, w.nsteps, 4, cudaMemcpyDeviceToHost, s));
  T2_CUDA(cudaStreamSynchronize(s));
  const int n = n_steps_host[0];
  if (n < 1 || n > max_steps) return fail(T2_ERR_CUDA, "infer_host: decoder reported %d steps", n);
  // frames beyond each row's length are zeroed (lengths mask); (B, 80, n) rows -> host rows of pitch max_steps
  T2PostnetArgs pa; memset(&pa, 0, sizeof(pa));
  pa.mel = w.mel; pa.mel_batch_stride = (long)max_steps * kMel; pa.lengths = w.lens; pa.add_residual = 1; pa.B = B; pa.T = n;
  pa.mel_post = w.post; pa.ws = w.sub; pa.ws_bytes = w.sub_bytes;
  T2_TRY(postnet_forward(m, &pa, s, ragged));
  T2_CUDA(cudaMemcpy2DAsync(mel_post_host, (size_t)max_steps * 4, w.post, (size_t)n * 4, (size_t)n * 4, (size_t)B * kMel,
                            cudaMemcpyDeviceToHost, s));
  if (n < max_steps) {   // frames past the last step: zeros
    float* tail = w.post + (size_t)B * kMel * n;
    T2_CUDA(cudaMemsetAsync(tail, 0, (size_t)B * kMel * (max_steps - n) * 4, s));
    T2_CUDA(cudaMemcpy2DAsync(mel_post_host + n, (size_t)max_steps * 4, tail, (size_t)(max_steps - n) * 4,
                              (size_t)(max_steps - n) * 4, (size_t)B * kMel, cudaMemcpyDeviceToHost, s));
  }
  T2_CUDA(cudaMemcpyAsync(mel_lengths_host, w.lens, (size_t)B * 4, cudaMemcpyDeviceToHost, s));
  T2_CUDA(cudaStreamSynchronize(s));
  return T2_OK;
}

int t2_infer_host(T2Model* m, const int64_t* text_host, int32_t B, int32_t T_text, int32_t max_steps,
                  float gate_threshold, uint64_t seed, int32_t impl, float* mel_post_host,
                  int32_t* mel_lengths_host, int32_t* n_steps_host, void* ws, size_t ws_bytes, void* stream) {
  return infer_host(m, text_host, nullptr, B, T_text, max_steps, gate_threshold, seed, impl, mel_post_host, mel_lengths_host,
                    n_steps_host, ws, ws_bytes, (cudaStream_t)stream);
}

int t2_infer_host_lengths(T2Model* m, const T2InferArgs* a, void* stream) {
  if (!a) return fail(T2_ERR_INVALID, "infer_host_lengths: null args");
  if (!a->input_lengths_host) return fail(T2_ERR_INVALID, "infer_host_lengths: null input_lengths_host (use t2_infer_host)");
  return infer_host(m, a->text_host, a->input_lengths_host, a->B, a->T_text, a->max_steps, a->gate_threshold, a->seed, a->impl,
                    a->mel_post_host, a->mel_lengths_host, a->n_steps_host, a->ws, a->ws_bytes, (cudaStream_t)stream);
}

int t2_decoder_profile(const T2DecoderArgs* a, int64_t* out_host) {
  if (!a || !out_host) return fail(T2_ERR_INVALID, "decoder_profile: null argument");
  DecoderWs w;
  T2_TRY(decoder_ws_carve(a, &w));
  T2_CUDA(cudaDeviceSynchronize());
  T2_CUDA(cudaMemcpy(out_host, w.ctrl->prof, sizeof(long long) * 72, cudaMemcpyDeviceToHost));
  return T2_OK;
}

// ---- WaveGlow (waveglow.cu) ----
int t2_waveglow_create(T2WaveGlow** out, const T2WaveGlowConfig* cfg, const void* const* weights, int32_t n_weights,
                       void* stream) {
  return waveglow_create(out, cfg, weights, n_weights, (cudaStream_t)stream);
}
int t2_waveglow_refresh(T2WaveGlow* h, const void* const* weights, int32_t n_weights, void* stream) {
  return waveglow_refresh(h, weights, n_weights, (cudaStream_t)stream);
}
int t2_waveglow_destroy(T2WaveGlow* h) { return waveglow_destroy(h); }
size_t t2_waveglow_workspace_bytes(const T2WaveGlow*, int32_t B, int32_t T_mel) {
  return B > 0 && T_mel > 0 ? waveglow_ws_bytes(B, T_mel) : 0;
}
int t2_waveglow_infer(T2WaveGlow* h, const T2WaveGlowArgs* a, void* stream) {
  return waveglow_infer(h, a, (cudaStream_t)stream);
}
int t2_waveglow_infer_window(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, void* stream) {
  return waveglow_infer_window(h, a, (cudaStream_t)stream);
}
void t2_waveglow_window_halo(int32_t* left, int32_t* right) { waveglow_window_halo(left, right); }

// ---- WaveGlow denoiser, STFT and Griffin-Lim (denoiser.cu) ----
int t2_denoiser_create(T2Denoiser** out, const T2DenoiserConfig* cfg, const float* forward_basis,
                       const float* inverse_basis, void* stream) {
  return denoiser_create(out, cfg, forward_basis, inverse_basis, (cudaStream_t)stream);
}
int t2_denoiser_refresh(T2Denoiser* h, const float* forward_basis, const float* inverse_basis, void* stream) {
  return denoiser_refresh(h, forward_basis, inverse_basis, (cudaStream_t)stream);
}
int t2_denoiser_destroy(T2Denoiser* h) { return denoiser_destroy(h); }
int t2_denoiser_bias(T2Denoiser* h, const float* audio, int32_t n, float* bias_out, void* stream) {
  return denoiser_bias(h, audio, n, bias_out, (cudaStream_t)stream);
}
size_t t2_denoiser_workspace_bytes(const T2Denoiser*, int32_t B, int32_t n) {
  return B > 0 && n > 0 ? denoiser_ws_bytes(B, n) : 0;
}
int t2_denoiser_run(T2Denoiser* h, const T2DenoiserArgs* a, void* stream) {
  return denoiser_run(h, a, (cudaStream_t)stream);
}
int t2_denoiser_run_window(T2Denoiser* h, const T2DenoiserWindowArgs* a, void* stream) {
  return denoiser_run_window(h, a, (cudaStream_t)stream);
}
void t2_denoiser_window_halo(int32_t* left, int32_t* right) { denoiser_window_halo(left, right); }
size_t t2_stft_transform_workspace_bytes(const T2Denoiser*, int32_t B, int32_t n) {
  return B > 0 && n > 0 ? stft_ws_bytes(B, n, false) : 0;
}
int t2_stft_transform(T2Denoiser* h, const T2StftTransformArgs* a, void* stream) {
  return stft_transform(h, a, (cudaStream_t)stream);
}
size_t t2_stft_inverse_workspace_bytes(const T2Denoiser*, int32_t B, int32_t F) {
  return B > 0 && F >= 4 ? stft_ws_bytes(B, 256 * (F - 1), false) : 0;
}
int t2_stft_inverse(T2Denoiser* h, const T2StftInverseArgs* a, void* stream) {
  return stft_inverse(h, a, (cudaStream_t)stream);
}
size_t t2_griffin_lim_workspace_bytes(const T2Denoiser*, int32_t B, int32_t F) {
  return B > 0 && F >= 4 ? stft_ws_bytes(B, 256 * (F - 1), true) : 0;
}
int t2_griffin_lim(T2Denoiser* h, const T2GriffinLimArgs* a, void* stream) {
  return griffin_lim(h, a, (cudaStream_t)stream);
}

#ifdef T2_SELFTEST   // libt2b200_selftest.so only
int t2_selftest_mma_rate(int32_t M, int32_t N, int32_t reps, int32_t alternate_d, int64_t* out_host) {
  return mma_rate(M, N, reps, alternate_d, (long long*)out_host, 0);
}

int t2_selftest_mma_group(int32_t M, int32_t N, int32_t group, int32_t reps, int64_t* out_host) {
  return mma_group(M, N, group, reps, (long long*)out_host, 0);
}

int t2_selftest_umma(const float* A, const float* W, int32_t N, int32_t K, int32_t passes, float* C, void* stream) {
  return selftest_umma(A, W, N, K, passes, C, (cudaStream_t)stream);
}

int t2_selftest_event(const float* A, const float* W, const int32_t* consumers, int32_t n_consumers, int32_t K, float* C,
                      void* stream) {
  return selftest_event(A, W, consumers, n_consumers, K, C, (cudaStream_t)stream);
}

// C = op(A) . op(B) + beta C through the training path's tensor-core GEMM (gemm_tc.cu); batch > 1: strided batch
int t2_selftest_gemm_tc(int32_t ta, int32_t tb, int32_t M, int32_t N, int32_t K, const float* A, int64_t lda, const float* B,
                        int64_t ldb, float* C, int64_t ldc, float beta, int32_t batch, int64_t strideA, int64_t strideB,
                        int64_t strideC, void* stream) {
  static T2Model scratch_owner;            // only its GEMM scratch is used
  GemmTc g;
  g.ta = ta != 0; g.tb = tb != 0; g.M = M; g.N = N; g.K = K; g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
  g.beta = beta; g.batch = batch; g.strideA = strideA; g.strideB = strideB; g.strideC = strideC;
  return gemm_tc(&scratch_owner, (cudaStream_t)stream, g);
}
int t2_selftest_colsum(const float* X, int64_t ld, int64_t rows, int32_t cols, float* out, void* stream) {
  static T2Model scratch_owner;
  return colsum_f32(&scratch_owner, (cudaStream_t)stream, X, ld, rows, cols, out);
}
int t2_selftest_waveglow_state(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, int32_t n_launches, float* spect, float* hbuf,
                               float* acts, float* skip, float* aud, void* stream) {
  return waveglow_state(h, a, n_launches, spect, hbuf, acts, skip, aud, (cudaStream_t)stream);
}
#endif

}  // extern "C"
