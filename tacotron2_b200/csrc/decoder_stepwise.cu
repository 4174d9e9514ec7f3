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

__global__ void __launch_bounds__(256)
attention_row_kernel(const float* __restrict__ ah, const float* __restrict__ Wq,
                     const float* __restrict__ Wloc, const float* __restrict__ Wld,
                     const float* __restrict__ v, const float* __restrict__ pm,
                     const float* __restrict__ memory, const int32_t* __restrict__ mem_len,
                     float score_mask_value, float* __restrict__ aw, float* __restrict__ awc,
                     float* __restrict__ ctx, float* __restrict__ align_out, long align_stride_b,
                     int T, const int* skip_flag) {
  if (skip_flag && *skip_flag) return;
  extern __shared__ float sm[];
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

  // 1. processed query  q = W_q . ah[b]            (model.py:57)
  const float* ahb = ah + (long)b * kARnn;
  for (int d = warp; d < kAtt; d += 8) {
    const float* wr = Wq + (long)d * kARnn;
    float s = 0.f;
    for (int k = lane; k < kARnn; k += 32) s = fmaf(wr[k], ahb[k], s);
    s = warp_sum(s);
    if (lane == 0) q[d] = s;
  }
  for (int i = tid; i < kLocF * kAtt; i += 256) {      // transpose (128,32) -> [c][d]
    const int d = i / kLocF, c = i - d * kLocF;
    wld_t[c * kAtt + d] = Wld[i];
  }
  for (int i = tid; i < kLocF * 2 * kLocK; i += 256) wloc[i] = Wloc[i];
  const int half = (kLocK - 1) / 2;
  for (int i = tid; i < TP; i += 256) {
    const int j = i - half;
    const bool in = (j >= 0 && j < T);
    pad0[i] = in ? aw[(long)b * T + j] : 0.f;
    pad1[i] = in ? awc[(long)b * T + j] : 0.f;
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
  const int len = mem_len ? mem_len[b] : T;
  for (int j = warp; j < T; j += 8) {
    float part = 0.f;
#pragma unroll
    for (int r = 0; r < kAtt / 32; ++r) {
      const int d = lane + 32 * r;
      float pa = 0.f;
#pragma unroll
      for (int c = 0; c < kLocF; ++c) pa = fmaf(wld_t[c * kAtt + d], loc[c * T + j], pa);
      const float x = q[d] + pa + pm[((long)b * T + j) * kAtt + d];
      part = fmaf(v[d], tanhf(x), part);
    }
    part = warp_sum(part);
    if (lane == 0) e[j] = (j < len) ? part : score_mask_value;     // model.py:79-80
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
    aw[(long)b * T + j] = p;
    awc[(long)b * T + j] += p;                                     // model.py:365
    align_out[(long)b * align_stride_b + j] = p;
  }
  __syncthreads();
  // 5. context = aw . memory                                          (model.py:83-84)
  for (int col = tid; col < kEnc; col += 256) {
    const float* mp = memory + (long)b * T * kEnc + col;
    float s = 0.f;
    for (int j = 0; j < T; ++j) s = fmaf(e[j], mp[(long)j * kEnc], s);
    ctx[(long)b * kEnc + col] = s;
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

  // processed_memory = memory_layer(memory)                      (model.py:288)
  {
    GemmArgs g;
    g.seg[0] = {a->memory, kEnc, m->w[W_ATT_MEMORY], kEnc, kEnc};
    g.M = B * T; g.N = kAtt; g.C = w.pm; g.ldc = kAtt;
    T2_TRY(gemm_f32(g, s));
  }
  T2_CUDA(cudaFuncSetAttribute(attention_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)att_smem));
  const int* skip = &w.ctrl->all_done;
  const int pw_blocks = (B * kARnn + 255) / 256;
  const float p_att = m->cfg.p_attention_dropout, p_dec = m->cfg.p_decoder_dropout;

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
    {  // attention LSTMCell on [prenet ; context]              (model.py:352-354)
      GemmArgs g;
      g.nseg = 3;
      g.seg[0] = {x2, kPre, m->w[W_ARNN_WIH], kPre + kEnc, kPre};
      g.seg[1] = {w.ctx, kEnc, m->w[W_ARNN_WIH] + kPre, kPre + kEnc, kEnc};
      g.seg[2] = {w.ah, kARnn, m->w[W_ARNN_WHH], kARnn, kARnn};
      g.M = B; g.N = 4 * kARnn; g.C = w.gates; g.ldc = 4 * kARnn; g.bias = m->arnn_b;
      g.skip_flag = skip;
      T2_TRY(gemm_f32(g, s));
      const uint8_t* keep = (a->training && a->att_keep) ? a->att_keep + (long)t * B * kARnn : nullptr;
      const int ph = (a->training && !a->att_keep) ? 1 : 0;
      lstm_pointwise_kernel<<<pw_blocks, 256, 0, s>>>(w.gates, w.ah, w.ac, B, kARnn, keep, ph,
                                                      a->seed, t * 4 + 2, p_att, skip);
      T2_LAUNCH_CHECK();
    }
    attention_row_kernel<<<B, 256, att_smem, s>>>(
        w.ah, m->w[W_ATT_QUERY], m->w[W_ATT_LOC_CONV], m->w[W_ATT_LOC_DENSE], m->w[W_ATT_V], w.pm,
        a->memory, a->memory_lengths, a->score_mask_value, w.aw, w.awc, w.ctx,
        a->align + (long)t * T, (long)cap * T, T, skip);
    T2_LAUNCH_CHECK();
    {  // decoder LSTMCell on [attention_hidden ; context]        (model.py:366-369)
      GemmArgs g;
      g.nseg = 3;
      g.seg[0] = {w.ah, kARnn, m->w[W_DRNN_WIH], kARnn + kEnc, kARnn};
      g.seg[1] = {w.ctx, kEnc, m->w[W_DRNN_WIH] + kARnn, kARnn + kEnc, kEnc};
      g.seg[2] = {w.dh, kDRnn, m->w[W_DRNN_WHH], kDRnn, kDRnn};
      g.M = B; g.N = 4 * kDRnn; g.C = w.gates; g.ldc = 4 * kDRnn; g.bias = m->drnn_b;
      g.skip_flag = skip;
      T2_TRY(gemm_f32(g, s));
      const uint8_t* keep = (a->training && a->dec_keep) ? a->dec_keep + (long)t * B * kDRnn : nullptr;
      const int ph = (a->training && !a->dec_keep) ? 1 : 0;
      lstm_pointwise_kernel<<<pw_blocks, 256, 0, s>>>(w.gates, w.dh, w.dc, B, kDRnn, keep, ph,
                                                      a->seed, t * 4 + 3, p_dec, skip);
      T2_LAUNCH_CHECK();
    }
    {  // linear_projection + gate_layer on [decoder_hidden ; context]   (model.py:373-378)
      GemmArgs g;
      g.nseg = 2;
      g.seg[0] = {w.dh, kDRnn, m->projgate_w, kDRnn + kEnc, kDRnn};
      g.seg[1] = {w.ctx, kEnc, m->projgate_w + kDRnn, kDRnn + kEnc, kEnc};
      g.M = B; g.N = kMel + 1; g.C = w.proj; g.ldc = kMel + 1; g.bias = m->projgate_b;
      g.skip_flag = skip;
      T2_TRY(gemm_f32(g, s));
    }
    emit_kernel<<<1, 256, 0, s>>>(w.proj, a->mel, a->gate, B, t, cap, infer ? 1 : 0,
                                  a->gate_threshold, w.ctrl, a->mel_lengths, a->n_steps);
    T2_LAUNCH_CHECK();
  }
  finalize_lengths_kernel<<<1, 256, 0, s>>>(w.ctrl, a->mel_lengths, a->n_steps, B);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
