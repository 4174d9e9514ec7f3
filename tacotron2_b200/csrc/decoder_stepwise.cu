// T2_IMPL_STEPWISE: the decoder loop as one short fp32 kernel sequence per step.
// Bring-up / cross-check implementation of Decoder.decode (model.py:340-379), Prenet
// (model.py:97-100) and the loops of Decoder.inference / Decoder.forward (model.py:381-454).
// The production implementation is the persistent kernel in decoder_persistent.cu; both are
// checked against the oracle by tests/test_decoder_gpu.py.
#include "decoder.h"
#include "gemm_f32.cuh"

namespace t2 {

// ---------------------------------------------------------------------------------------------
// LSTM pointwise: gates (B, 4H) [i f g o] (biases already added) -> c, h   (torch.nn.LSTMCell)
// ---------------------------------------------------------------------------------------------
__global__ void lstm_pointwise_kernel(const float* __restrict__ gates, float* __restrict__ h,
                                      float* __restrict__ c, int B, int H,
                                      const uint8_t* __restrict__ keep, int philox, uint64_t seed,
                                      uint32_t site, float p_drop, const int* skip_flag) {
  if (skip_flag && *skip_flag) return;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H, j = idx - b * H;
  const float* g = gates + (long)b * 4 * H;
  const float gi = 1.f / (1.f + expf(-g[j]));
  const float gf = 1.f / (1.f + expf(-g[H + j]));
  const float gg = tanhf(g[2 * H + j]);
  const float go = 1.f / (1.f + expf(-g[3 * H + j]));
  const float cn = gf * c[idx] + gi * gg;
  float hn = go * tanhf(cn);
  if (keep) hn = keep[idx] ? hn * (1.f / (1.f - p_drop)) : 0.f;
  else if (philox) hn = philox_keep(seed, site, idx, p_drop) ? hn * (1.f / (1.f - p_drop)) : 0.f;
  c[idx] = cn;
  h[idx] = hn;
}

// ---------------------------------------------------------------------------------------------
// Location-sensitive attention for one batch row per CTA (model.py:22-26, 43-86, 358-365)
// ---------------------------------------------------------------------------------------------
__device__ inline float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ inline float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Row b reads its previous / cumulative weights at aw_in + b * in_stride and awc_in + b * in_stride: the decoder's
// state arrays (in_stride = T) or the two channels of attention_weights_cat (B, 2, T) (in_stride = 2 T).  Every output
// may be null; aw_out / awc_out may be aw_in / awc_in.
struct AttnRowArgs {
  const float *Wq, *Wloc, *Wld, *v;
  const float* ah;                  // (B, 1024) query, or null (zero query)
  const float* pm;                  // (B, T, 128) processed memory, or null (zero)
  const float* memory;              // (B, T, 512); read only for ctx
  const int32_t* mem_len;           // (B) or null: positions j >= mem_len[b] are masked
  const uint8_t* mask;              // (B, T) or null: 1 = masked, as the reference's mask; replaces mem_len
  float score_mask_value;
  const float* aw_in; const float* awc_in; long in_stride;
  float* aw_out; float* awc_out;    // new weights; awc_in + new weights
  float* ctx;                       // (B, 512)
  float* align_out; long align_stride_b;
  float* energies_out;              // (B, T) energies before the mask
  float* loc_out;                   // (B, T, 128) location term
  int T;
  const int* skip_flag;
};

__global__ void __launch_bounds__(256) attention_row_kernel(AttnRowArgs a) {
  if (a.skip_flag && *a.skip_flag) return;
  extern __shared__ float sm[];
  const int T = a.T;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int TP = T + kLocK - 1;                       // padded length
  float* q = sm;                                       // 128
  float* wld_t = q + kAtt;                             // [32][128]  (c-major)
  float* wloc = wld_t + kLocF * kAtt;                  // [32][2][31]
  float* pad0 = wloc + kLocF * 2 * kLocK;              // [TP] previous weights, zero padded
  float* pad1 = pad0 + TP;                             // [TP] cumulative weights
  float* loc = pad1 + TP;                              // [32][T]
  float* e = loc + kLocF * T;                          // [T]
  float* red = e + T;                                  // [32]

  // 1. processed query  q = W_q . ah[b]            (model.py:57); no query: the location term alone
  const float* ahb = a.ah + (long)b * kARnn;
  for (int d = warp; d < kAtt; d += 8) {
    const float* wr = a.Wq + (long)d * kARnn;
    float s = 0.f;
    if (a.ah)
      for (int k = lane; k < kARnn; k += 32) s = fmaf(wr[k], ahb[k], s);
    s = warp_sum(s);
    if (lane == 0) q[d] = s;
  }
  for (int i = tid; i < kLocF * kAtt; i += 256) {      // transpose (128,32) -> [c][d]
    const int d = i / kLocF, c = i - d * kLocF;
    wld_t[c * kAtt + d] = a.Wld[i];
  }
  for (int i = tid; i < kLocF * 2 * kLocK; i += 256) wloc[i] = a.Wloc[i];
  const int half = (kLocK - 1) / 2;
  for (int i = tid; i < TP; i += 256) {
    const int j = i - half;
    const bool in = (j >= 0 && j < T);
    pad0[i] = in ? a.aw_in[(long)b * a.in_stride + j] : 0.f;
    pad1[i] = in ? a.awc_in[(long)b * a.in_stride + j] : 0.f;
  }
  __syncthreads();
  // 2. location conv (2 -> 32 channels, k = 31, zero padding 15)     (model.py:23)
  for (int i = tid; i < kLocF * T; i += 256) {
    const int c = i / T, j = i - c * T;
    const float* w0 = wloc + c * 2 * kLocK;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kLocK; ++k) s = fmaf(w0[k], pad0[j + k], s);
#pragma unroll
    for (int k = 0; k < kLocK; ++k) s = fmaf(w0[kLocK + k], pad1[j + k], s);
    loc[i] = s;
  }
  __syncthreads();
  // 3. energies  e_j = v . tanh(q + W_ld loc_j + pm_j)               (model.py:24-25, 58-60)
  const int len = a.mem_len ? a.mem_len[b] : T;
  for (int j = warp; j < T; j += 8) {
    float part = 0.f;
#pragma unroll
    for (int r = 0; r < kAtt / 32; ++r) {
      const int d = lane + 32 * r;
      float pa = 0.f;
#pragma unroll
      for (int c = 0; c < kLocF; ++c) pa = fmaf(wld_t[c * kAtt + d], loc[c * T + j], pa);
      if (a.loc_out) a.loc_out[((long)b * T + j) * kAtt + d] = pa;              // LocationLayer.forward
      const float x = q[d] + pa + (a.pm ? a.pm[((long)b * T + j) * kAtt + d] : 0.f);
      part = fmaf(a.v[d], tanhf(x), part);
    }
    part = warp_sum(part);
    if (lane == 0) {
      if (a.energies_out) a.energies_out[(long)b * T + j] = part;               // get_alignment_energies
      const bool masked = a.mask ? a.mask[(long)b * T + j] != 0 : j >= len;
      e[j] = masked ? a.score_mask_value : part;                                 // model.py:79-80
    }
  }
  __syncthreads();
  // 4. softmax over T                                                 (model.py:82)
  float mx = -INFINITY;
  for (int j = tid; j < T; j += 256) mx = fmaxf(mx, e[j]);
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < T; j += 256) {
    const float p = expf(e[j] - mx);
    e[j] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.f / sum;
  for (int j = tid; j < T; j += 256) {
    const float p = e[j] * inv;
    e[j] = p;
    if (a.aw_out) a.aw_out[(long)b * T + j] = p;
    if (a.awc_out) a.awc_out[(long)b * T + j] = a.awc_in[(long)b * a.in_stride + j] + p;   // model.py:365
    if (a.align_out) a.align_out[(long)b * a.align_stride_b + j] = p;
  }
  __syncthreads();
  // 5. context = aw . memory                                          (model.py:83-84)
  if (!a.ctx) return;
  for (int col = tid; col < kEnc; col += 256) {
    const float* mp = a.memory + (long)b * T * kEnc + col;
    float s = 0.f;
    for (int j = 0; j < T; ++j) s = fmaf(e[j], mp[(long)j * kEnc], s);
    a.ctx[(long)b * kEnc + col] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// emit: scratch projection (B, 81) -> mel_out / gate_out, stop latch (model.py:443-447)
// ---------------------------------------------------------------------------------------------
__global__ void emit_kernel(const float* __restrict__ proj, float* __restrict__ mel_out,
                            float* __restrict__ gate_out, int B, int t, int T_cap, int infer,
                            float gate_threshold, DecoderCtrl* ctrl, int32_t* mel_lengths,
                            int32_t* n_steps) {
  if (ctrl->all_done) return;
  __shared__ int s_live;
  if (threadIdx.x == 0) s_live = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < B * kMel; i += blockDim.x) {
    const int b = i / kMel, c = i - b * kMel;
    mel_out[((long)b * T_cap + t) * kMel + c] = proj[b * (kMel + 1) + c];
  }
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float g = proj[b * (kMel + 1) + kMel];
    gate_out[(long)b * T_cap + t] = g;
    if (infer) {
      int done = ctrl->done[b];
      if (!done && (1.f / (1.f + expf(-g))) > gate_threshold) {   // predicate of model.py:443
        done = 1;
        ctrl->done[b] = 1;
        mel_lengths[b] = t + 1;
      }
      if (!done) atomicAdd(&s_live, 1);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *n_steps = t + 1;
    if (infer && s_live == 0) ctrl->all_done = 1;
  }
}

__global__ void finalize_lengths_kernel(DecoderCtrl* ctrl, int32_t* mel_lengths,
                                        const int32_t* n_steps, int B) {
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    if (!ctrl->done[b]) mel_lengths[b] = *n_steps;
}

size_t stepwise_attention_smem(int T) {
  return sizeof(float) * (kAtt + kLocF * kAtt + kLocF * 2 * kLocK + 2 * (T + kLocK - 1) +
                          kLocF * T + T + 32);
}

static int attention_smem_opt_in(size_t att_smem) {
  T2_CUDA(cudaFuncSetAttribute(attention_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)att_smem));
  return T2_OK;
}

// workspace of the stepwise decoder
struct StepwiseWs {
  float* pm;               // processed_memory (B, T, 128)          model.py:288
  char* state_begin; size_t state_bytes;   // zero-initialised block (model.py:258-284):
  float *ah, *ac, *dh, *dc;                // (B, 1024) each
  float* ctx;              // (B, 512)
  float *aw, *awc;         // (B, T)
  float *x1, *x2;          // prenet activations (B, 256)
  float* gates;            // (B, 4096)
  float* proj;             // (B, 81)
  DecoderCtrl* ctrl;
};
static void stepwise_ws_layout(Carve& c, int B, int T, StepwiseWs* w) {
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
}
size_t stepwise_ws_bytes(int B, int T) {
  Carve c(nullptr, kDecoderWsAlign);
  StepwiseWs w;
  stepwise_ws_layout(c, B, T, &w);
  return c.bytes();
}

// ---------------------------------------------------------------------------------------------
// one decoder step (Decoder.decode, model.py:340-379) after the prenet, on the state arrays `st`, in place
// ---------------------------------------------------------------------------------------------
int decoder_step(T2Model* m, const StepState& st, const StepIo& io, cudaStream_t s) {
  const int B = io.B, T = io.T;
  const int pw_blocks = (B * kARnn + 255) / 256;
  const float p_att = m->cfg.p_attention_dropout, p_dec = m->cfg.p_decoder_dropout;
  {  // attention LSTMCell on [prenet ; context]              (model.py:352-354)
    GemmArgs g;
    g.nseg = 3;
    g.seg[0] = {io.x2, kPre, m->w[W_ARNN_WIH], kPre + kEnc, kPre};
    g.seg[1] = {st.ctx, kEnc, m->w[W_ARNN_WIH] + kPre, kPre + kEnc, kEnc};
    g.seg[2] = {st.ah, kARnn, m->w[W_ARNN_WHH], kARnn, kARnn};
    g.M = B; g.N = 4 * kARnn; g.C = io.gates; g.ldc = 4 * kARnn; g.bias = m->arnn_b;
    g.skip_flag = io.skip;
    T2_TRY(gemm_f32(g, s));
    const uint8_t* keep = io.training ? io.att_keep : nullptr;
    const int ph = (io.training && !io.att_keep) ? 1 : 0;
    lstm_pointwise_kernel<<<pw_blocks, 256, 0, s>>>(io.gates, st.ah, st.ac, B, kARnn, keep, ph,
                                                    io.seed, io.site + 2, p_att, io.skip);
    T2_LAUNCH_CHECK();
  }
  {  // attention (model.py:358-365): new weights, cumulative update, context
    AttnRowArgs a;
    a.Wq = m->w[W_ATT_QUERY]; a.Wloc = m->w[W_ATT_LOC_CONV]; a.Wld = m->w[W_ATT_LOC_DENSE]; a.v = m->w[W_ATT_V];
    a.ah = st.ah; a.pm = io.pm; a.memory = io.memory; a.mem_len = io.mem_len; a.mask = io.mask;
    a.score_mask_value = io.score_mask_value;
    a.aw_in = st.aw; a.awc_in = st.awc; a.in_stride = T;
    a.aw_out = st.aw; a.awc_out = st.awc; a.ctx = st.ctx;
    a.align_out = io.align_out; a.align_stride_b = io.align_stride_b;
    a.energies_out = nullptr; a.loc_out = nullptr;
    a.T = T; a.skip_flag = io.skip;
    attention_row_kernel<<<B, 256, stepwise_attention_smem(T), s>>>(a);
    T2_LAUNCH_CHECK();
  }
  {  // decoder LSTMCell on [attention_hidden ; context]        (model.py:366-369)
    GemmArgs g;
    g.nseg = 3;
    g.seg[0] = {st.ah, kARnn, m->w[W_DRNN_WIH], kARnn + kEnc, kARnn};
    g.seg[1] = {st.ctx, kEnc, m->w[W_DRNN_WIH] + kARnn, kARnn + kEnc, kEnc};
    g.seg[2] = {st.dh, kDRnn, m->w[W_DRNN_WHH], kDRnn, kDRnn};
    g.M = B; g.N = 4 * kDRnn; g.C = io.gates; g.ldc = 4 * kDRnn; g.bias = m->drnn_b;
    g.skip_flag = io.skip;
    T2_TRY(gemm_f32(g, s));
    const uint8_t* keep = io.training ? io.dec_keep : nullptr;
    const int ph = (io.training && !io.dec_keep) ? 1 : 0;
    lstm_pointwise_kernel<<<pw_blocks, 256, 0, s>>>(io.gates, st.dh, st.dc, B, kDRnn, keep, ph,
                                                    io.seed, io.site + 3, p_dec, io.skip);
    T2_LAUNCH_CHECK();
  }
  {  // linear_projection + gate_layer on [decoder_hidden ; context]   (model.py:373-378)
    GemmArgs g;
    g.nseg = 2;
    g.seg[0] = {st.dh, kDRnn, m->projgate_w, kDRnn + kEnc, kDRnn};
    g.seg[1] = {st.ctx, kEnc, m->projgate_w + kDRnn, kDRnn + kEnc, kEnc};
    g.M = B; g.N = kMel + 1; g.C = io.proj; g.ldc = kMel + 1; g.bias = m->projgate_b;
    g.skip_flag = io.skip;
    T2_TRY(gemm_f32(g, s));
  }
  return T2_OK;
}

// ---------------------------------------------------------------------------------------------
// host orchestration
// ---------------------------------------------------------------------------------------------
int decoder_run_stepwise(T2Model* m, const T2DecoderArgs* a, cudaStream_t s) {
  const int B = a->B, T = a->T_enc, cap = a->n_steps_cap;
  const bool infer = a->mode == T2_MODE_INFER;
  const size_t att_smem = stepwise_attention_smem(T);
  if (att_smem > 200 * 1024) return fail(T2_ERR_INVALID, "T_enc=%d too long for the stepwise attention kernel (at most 1282)", T);
  Carve c(a->ws, kDecoderWsAlign);
  StepwiseWs w;
  stepwise_ws_layout(c, B, T, &w);
  T2_CUDA(cudaMemsetAsync(w.state_begin, 0, w.state_bytes, s));   // model.py:258-284 (zeros)
  T2_CUDA(cudaMemsetAsync(w.ctrl, 0, sizeof(DecoderCtrl), s));

  T2_TRY(processed_memory(m, a->memory, B, T, w.pm, s));
  T2_TRY(attention_smem_opt_in(att_smem));
  const int* skip = &w.ctrl->all_done;
  const StepState st{w.ah, w.ac, w.dh, w.dc, w.aw, w.awc, w.ctx};

  for (int t = 0; t < cap; ++t) {
    const float* x2;
    if (infer) {
      // Prenet on the fed-back frame (model.py:436, 449); step 0 consumes the go frame (:430)
      GemmArgs g;
      const float* prev = (t == 0) ? m->zeros : a->mel + (long)(t - 1) * kMel;
      g.seg[0] = {prev, (t == 0) ? 0L : (long)cap * kMel, m->w[W_PRENET0], kMel, kMel};
      g.M = B; g.N = kPre; g.C = w.x1; g.ldc = kPre; g.act = ACT_RELU; g.p_drop = 0.5f;
      if (a->prenet_keep) { g.keep = a->prenet_keep + ((long)t * 2 + 0) * B * kPre; g.ldkeep = kPre; }
      else { g.philox = 1; g.seed = a->seed; g.site = t * 4 + 0; g.row_seeds = a->row_seeds; }
      g.skip_flag = skip;
      T2_TRY(gemm_f32(g, s));
      GemmArgs h;
      h.seg[0] = {w.x1, kPre, m->w[W_PRENET1], kPre, kPre};
      h.M = B; h.N = kPre; h.C = w.x2; h.ldc = kPre; h.act = ACT_RELU; h.p_drop = 0.5f;
      if (a->prenet_keep) { h.keep = a->prenet_keep + ((long)t * 2 + 1) * B * kPre; h.ldkeep = kPre; }
      else { h.philox = 1; h.seed = a->seed; h.site = t * 4 + 1; h.row_seeds = a->row_seeds; }
      h.skip_flag = skip;
      T2_TRY(gemm_f32(h, s));
      x2 = w.x2;
    } else {
      x2 = a->teacher_prenet + (long)t * B * kPre;
    }
    StepIo io;
    io.x2 = x2; io.memory = a->memory; io.pm = w.pm; io.mem_len = a->memory_lengths;
    io.score_mask_value = a->score_mask_value; io.B = B; io.T = T;
    io.training = a->training;
    io.att_keep = a->att_keep ? a->att_keep + (long)t * B * kARnn : nullptr;
    io.dec_keep = a->dec_keep ? a->dec_keep + (long)t * B * kDRnn : nullptr;
    io.seed = a->seed; io.site = t * 4; io.gates = w.gates; io.proj = w.proj;
    io.align_out = a->align + (long)t * T; io.align_stride_b = (long)cap * T; io.skip = skip;
    T2_TRY(decoder_step(m, st, io, s));
    emit_kernel<<<1, 256, 0, s>>>(w.proj, a->mel, a->gate, B, t, cap, infer ? 1 : 0,
                                  a->gate_threshold, w.ctrl, a->mel_lengths, a->n_steps);
    T2_LAUNCH_CHECK();
  }
  finalize_lengths_kernel<<<1, 256, 0, s>>>(w.ctrl, a->mel_lengths, a->n_steps, B);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

// processed_memory = memory_layer(memory)                      (model.py:288)
int processed_memory(T2Model* m, const float* memory, int B, int T, float* out, cudaStream_t s) {
  GemmArgs g;
  g.seg[0] = {memory, kEnc, m->w[W_ATT_MEMORY], kEnc, kEnc};
  g.M = B * T; g.N = kAtt; g.C = out; g.ldc = kAtt;
  return gemm_f32(g, s);
}

// ---------------------------------------------------------------------------------------------
// t2_decoder_step: one decode() on the caller's state
// ---------------------------------------------------------------------------------------------
__global__ void split_proj_kernel(const float* __restrict__ proj, float* __restrict__ mel, float* __restrict__ gate, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * (kMel + 1)) return;
  const int b = i / (kMel + 1), c = i - b * (kMel + 1);
  if (c < kMel) mel[b * kMel + c] = proj[i];
  else gate[b] = proj[i];
}

static void step_ws_layout(Carve& c, int B, float** gates, float** proj) {
  *gates = c.take<float>((size_t)B * 4 * kARnn);
  *proj = c.take<float>((size_t)B * (kMel + 1));
}
size_t decoder_step_ws_bytes(int B) {
  Carve c(nullptr);
  float *g, *p;
  step_ws_layout(c, B, &g, &p);
  return c.bytes();
}

int decoder_step_run(T2Model* m, const T2DecoderStepArgs* a, cudaStream_t s) {
  const int B = a->B, T = a->T_enc;
  T2_TRY(attention_smem_opt_in(stepwise_attention_smem(T)));
  float *gates, *proj;
  Carve c(a->ws);
  step_ws_layout(c, B, &gates, &proj);
  const StepState st{a->attention_hidden, a->attention_cell, a->decoder_hidden, a->decoder_cell, a->attention_weights,
                     a->attention_weights_cum, a->attention_context};
  StepIo io;
  io.x2 = a->decoder_input; io.memory = a->memory; io.pm = a->processed_memory; io.mask = a->mask;
  io.score_mask_value = a->score_mask_value; io.B = B; io.T = T;
  io.training = a->training; io.att_keep = a->att_keep; io.dec_keep = a->dec_keep;
  io.seed = a->seed; io.site = 0;                  // the keys of step 0 of decoder_run_stepwise
  io.gates = gates; io.proj = proj;
  T2_TRY(decoder_step(m, st, io, s));
  split_proj_kernel<<<(B * (kMel + 1) + 255) / 256, 256, 0, s>>>(proj, a->mel, a->gate, B);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

// ---------------------------------------------------------------------------------------------
// t2_attention_forward: Attention.forward / get_alignment_energies / LocationLayer.forward
// ---------------------------------------------------------------------------------------------
int attention_forward(T2Model* m, const T2AttentionArgs* a, cudaStream_t s) {
  const int T = a->T_enc;
  T2_TRY(attention_smem_opt_in(stepwise_attention_smem(T)));
  AttnRowArgs r;
  r.Wq = m->w[W_ATT_QUERY]; r.Wloc = m->w[W_ATT_LOC_CONV]; r.Wld = m->w[W_ATT_LOC_DENSE]; r.v = m->w[W_ATT_V];
  r.ah = a->query; r.pm = a->processed_memory; r.memory = a->memory; r.mem_len = nullptr; r.mask = a->mask;
  r.score_mask_value = a->score_mask_value;
  r.aw_in = a->attention_weights_cat; r.awc_in = a->attention_weights_cat + T; r.in_stride = 2L * T;
  r.aw_out = a->weights; r.awc_out = nullptr; r.ctx = a->context; r.align_out = nullptr; r.align_stride_b = 0;
  r.energies_out = a->energies; r.loc_out = a->location;
  r.T = T; r.skip_flag = nullptr;
  attention_row_kernel<<<a->B, 256, stepwise_attention_smem(T), s>>>(r);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
