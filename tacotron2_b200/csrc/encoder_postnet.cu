// Encoder (model.py:149-201) and Postnet (model.py:103-146) forwards: the evaluation-mode conv stacks on the tensor-core
// conv engine, the training-mode ones handed to train_layers.cu, and the encoder BiLSTM.
#include "conv_tc.h"
#include "gemm_f32.cuh"
#include "train_layers.h"
#include "model.h"

namespace t2 {

// One time step of both directions of the encoder BiLSTM (model.py:169-171, 180-188).
// grid (16 unit blocks, 2 directions, batch chunks of 64); 256 threads = 64 rows x 4 unit groups.
__global__ void __launch_bounds__(256)
enc_lstm_step_kernel(const float* __restrict__ gin,   // (B, T, 2048) W_ih x + b, fwd | reverse
                     const float* __restrict__ whh_f, const float* __restrict__ whh_r,
                     const float* __restrict__ h_in, float* __restrict__ h_out,  // (2, B, 256)
                     float* __restrict__ c,                                        // (2, B, 256)
                     float* __restrict__ memory,                                   // (B, T, 512)
                     const int32_t* __restrict__ lengths, int B, int T, int step) {
  extern __shared__ float sm[];
  float* ws = sm;                    // [64 rows][256]
  float* hs = sm + 64 * kEncH;       // [64][257]
  const int ub = blockIdx.x, dir = blockIdx.y, b0 = blockIdx.z * 64;
  const int tid = threadIdx.x;
  const int t = dir == 0 ? step : T - 1 - step;
  const float* whh = dir == 0 ? whh_f : whh_r;
  // smem row r = ul*4 + gate  <-  weight_hh row gate*256 + (ub*16 + ul)
  for (int i = tid; i < 64 * kEncH / 4; i += 256) {
    const int r = i / (kEncH / 4), k4 = i % (kEncH / 4);
    const int ul = r >> 2, gate = r & 3;
    reinterpret_cast<float4*>(ws)[i] =
        reinterpret_cast<const float4*>(whh + ((long)gate * kEncH + ub * 16 + ul) * kEncH)[k4];
  }
  for (int i = tid; i < 64 * kEncH; i += 256) {
    const int bl = i / kEncH, k = i % kEncH;
    hs[bl * (kEncH + 1) + k] = (b0 + bl < B) ? h_in[((long)dir * B + b0 + bl) * kEncH + k] : 0.f;
  }
  __syncthreads();
  const int bl = tid & 63, ug = tid >> 6;
  const int b = b0 + bl;
  float acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int g = 0; g < 4; ++g) acc[u][g] = 0.f;
  const float* hrow = hs + bl * (kEncH + 1);
  const float* wbase = ws + (ug * 16) * kEncH;
  for (int k = 0; k < kEncH; ++k) {
    const float hv = hrow[k];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int g = 0; g < 4; ++g) acc[u][g] = fmaf(wbase[(u * 4 + g) * kEncH + k], hv, acc[u][g]);
  }
  if (b >= B) return;
  const bool valid = lengths == nullptr || t < lengths[b];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int unit = ub * 16 + ug * 4 + u;
    const float* gp = gin + ((long)b * T + t) * (8 * kEncH) + dir * 4 * kEncH;
    const long si = ((long)dir * B + b) * kEncH + unit;
    float hn = hrow[unit], cn = c[si];
    if (valid) {
      const float gi = 1.f / (1.f + expf(-(acc[u][0] + gp[unit])));
      const float gf = 1.f / (1.f + expf(-(acc[u][1] + gp[kEncH + unit])));
      const float gg = tanhf(acc[u][2] + gp[2 * kEncH + unit]);
      const float go = 1.f / (1.f + expf(-(acc[u][3] + gp[3 * kEncH + unit])));
      cn = gf * cn + gi * gg;
      hn = go * tanhf(cn);
      c[si] = cn;
    }
    h_out[si] = hn;
    memory[((long)b * T + t) * kEnc + dir * kEncH + unit] = valid ? hn : 0.f;
  }
}

// Persistent variant of the recurrence: ONE cooperative launch runs all T steps of both directions.
// 128 CTAs = 2 directions x 64 unit blocks of 4 hidden units (16 gate rows); the CTA's W_hh slice stays
// in shared memory for the whole sequence, h is exchanged through a double-buffered global array and a
// grid-wide barrier (monotonic counter) per step.  256 threads = 64 batch rows x 4 units; each thread
// owns the 4 gates of ONE (row, unit) pair, so the cell state lives in a register.
struct EncLstmCtrl { unsigned int bar_count; unsigned int pad_[3]; };

__global__ void __launch_bounds__(256, 1)
enc_lstm_persistent_kernel(const float* __restrict__ gin, const float* __restrict__ whh_f,
                           const float* __restrict__ whh_r, float* __restrict__ hbuf,   // (2 buffers, 2 dirs, B, 256)
                           float* __restrict__ memory, const int32_t* __restrict__ lengths, int B, int T,
                           EncLstmCtrl* ctrl, float* __restrict__ st_gates, float* __restrict__ st_c) {
  extern __shared__ float sm[];
  float* ws = sm;                        // [64 k4][16 rows][4]   (row = gate*4 + unit_local)
  float* hs = sm + kEncH * 16;           // [64 k4][64 batch][4]
  const int cta = blockIdx.x, dir = cta >> 6, ub = cta & 63;
  const int tid = threadIdx.x;
  const float* whh = dir == 0 ? whh_f : whh_r;
  for (int i = tid; i < 16 * (kEncH / 4); i += 256) {
    const int r = i / (kEncH / 4), k4 = i % (kEncH / 4);
    const int gate = r >> 2, ul = r & 3;
    const float4 v = reinterpret_cast<const float4*>(whh + ((long)gate * kEncH + ub * 4 + ul) * kEncH)[k4];
    reinterpret_cast<float4*>(ws)[k4 * 16 + r] = v;
  }
  const int b = tid & 63, ul = tid >> 6;             // batch row, local unit
  const int unit = ub * 4 + ul;
  float c = 0.f, hprev = 0.f;
  unsigned int target = 0;
  __syncthreads();
  for (int step = 0; step < T; ++step) {
    const int t = dir == 0 ? step : T - 1 - step;
    const float* hin = hbuf + ((long)(step & 1) * 2 + dir) * B * kEncH;
    float* hout = hbuf + ((long)((step + 1) & 1) * 2 + dir) * B * kEncH;
    // gate pre-activations from the input projection (issued first: their latency hides behind the GEMV)
    float gi4[4] = {0.f, 0.f, 0.f, 0.f};
    const bool live = b < B;
    const bool valid = live && (lengths == nullptr || t < lengths[b]);
    if (live) {
      const float* gp = gin + ((long)b * T + t) * (8 * kEncH) + dir * 4 * kEncH + unit;
#pragma unroll
      for (int g = 0; g < 4; ++g) gi4[g] = __ldg(gp + g * kEncH);
    }
    for (int i = tid; i < 64 * (kEncH / 4); i += 256) {       // h_(t-1) of all rows -> [k4][b][4]
      const int bb = i / (kEncH / 4), k4 = i % (kEncH / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (bb < B) v = __ldcg(reinterpret_cast<const float4*>(hin + (long)bb * kEncH) + k4);
      reinterpret_cast<float4*>(hs)[k4 * 64 + bb] = v;
    }
    __syncthreads();
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
    for (int k4 = 0; k4 < kEncH / 4; ++k4) {
      const float4 hv = reinterpret_cast<const float4*>(hs)[k4 * 64 + b];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const float4 wv = reinterpret_cast<const float4*>(ws)[k4 * 16 + g * 4 + ul];
        acc[g] = fmaf(wv.x, hv.x, acc[g]); acc[g] = fmaf(wv.y, hv.y, acc[g]);
        acc[g] = fmaf(wv.z, hv.z, acc[g]); acc[g] = fmaf(wv.w, hv.w, acc[g]);
      }
    }
    if (live) {
      float hn = hprev;
      if (valid) {
        const float gi = 1.f / (1.f + expf(-(acc[0] + gi4[0])));
        const float gf = 1.f / (1.f + expf(-(acc[1] + gi4[1])));
        const float gg = tanhf(acc[2] + gi4[2]);
        const float go = 1.f / (1.f + expf(-(acc[3] + gi4[3])));
        c = gf * c + gi * gg;
        hn = go * tanhf(c);
        if (st_gates) {   // training stash: gate activations in the layout of gin
          float* sg = st_gates + ((long)b * T + t) * (8 * kEncH) + dir * 4 * kEncH + unit;
          sg[0] = gi; sg[kEncH] = gf; sg[2 * kEncH] = gg; sg[3 * kEncH] = go;
        }
      }
      if (st_c) st_c[((long)b * T + t) * kEnc + dir * kEncH + unit] = c;
      hprev = hn;
      hout[(long)b * kEncH + unit] = hn;
      memory[((long)b * T + t) * kEnc + dir * kEncH + unit] = valid ? hn : 0.f;
    }
    // grid barrier (monotonic counter, red.release / ld.acquire)
    __syncthreads();
    target += gridDim.x;
    if (tid == 0) {
      __threadfence();
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(&ctrl->bar_count) : "memory");
      const unsigned long long t0 = clock64();
      while (true) {
        unsigned int cnt;
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cnt) : "l"(&ctrl->bar_count) : "memory");
        if ((int)(cnt - target) >= 0) break;
        if (clock64() - t0 > (1ull << 32)) __trap();
      }
    }
    __syncthreads();
  }
}

// ---- host side ----------------------------------------------------------------------------------
// Two conv paths: evaluation-mode forwards without a stash run on the tensor-core inference convs (conv_tc.cu); every
// training-mode forward and every forward under autograd (a stash) runs on the training conv stack (train_layers.cu).
// A call runs one of them, so the inference planes and the training stack share their bytes of the workspace.
struct EncoderWs {
  float* gin;              // (B, T, 2048) LSTM input projections, forward | reverse
  float* h;                // (2, 2, B, 256): two h buffers (read / write) of both directions
  float* c;                // (2, B, 256)
  float *scale, *shift;    // (2048) folded BatchNorm / bias
  EncLstmCtrl* lctrl;
  __half *pl0, *pl1;       // tensor-core activation planes
  void* train;             // the training conv stack without a stash (on the planes' bytes)
};
static void encoder_ws_layout(Carve& c, int B, int T, EncoderWs* w) {
  w->gin = c.take<float>((size_t)B * T * 8 * kEncH);
  w->h = c.take<float>((size_t)2 * 2 * B * kEncH);
  w->c = c.take<float>((size_t)2 * B * kEncH);
  w->scale = c.take<float>(8 * kEncH); w->shift = c.take<float>(8 * kEncH);
  w->lctrl = c.take<EncLstmCtrl>(1);
  Carve planes = c;
  w->pl0 = planes.take<__half>(tc_planes_bytes(B, T, kEnc) / sizeof(__half));
  w->pl1 = planes.take<__half>(tc_planes_bytes(B, T, kEnc) / sizeof(__half));
  w->train = c.take<char>(encoder_convs_train_ws_bytes(B, T));
  if (planes.off > c.off) c.off = planes.off;
}
size_t encoder_ws_bytes(int B, int T) { Carve c(nullptr); EncoderWs w; encoder_ws_layout(c, B, T, &w); return c.bytes(); }

// per_row (t2_encoder_infer): each row b is encoded as its first lengths[b] symbols alone -- the inputs at t >= lengths[b]
// and every conv layer's outputs there are zero, the padding the row has at T = lengths[b].  Otherwise lengths only
// masks the BiLSTM (pack_padded_sequence, model.py:180-188) and the convolutions see the padded inputs as the
// reference's do.
int encoder_forward(T2Model* m, const T2EncoderArgs* a, cudaStream_t s, bool per_row) {
  const int B = a->B, T = a->T;
  if (B <= 0 || T <= 0) return fail(T2_ERR_INVALID, "encoder: empty batch");
  if (a->ws_bytes < encoder_ws_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "encoder workspace too small");
  const bool persistent = B <= 64 && m->sm_count >= 128;      // the BiLSTM as one cooperative launch
  if (a->stash && !persistent)
    return fail(T2_ERR_UNSUPPORTED, "encoder: the training stash needs B <= 64 and >= 128 SMs (persistent BiLSTM kernel)");
  Carve cv(a->ws);
  EncoderWs w;
  encoder_ws_layout(cv, B, T, &w);
  float* st_gates = nullptr; float* st_c = nullptr;
  const int32_t* conv_len = per_row ? a->lengths : nullptr;

  if (a->training || a->stash) {
    // training conv stack (fp32), then W_ih x + b_ih + b_hh for every time step and both directions
    const float* xl = nullptr;
    T2_TRY(encoder_convs_train(m, a, w.train, s, &xl, &st_gates, &st_c));
    GemmArgs g;
    g.seg[0] = {xl, kEnc, m->enc_lstm_wih, kEnc, kEnc};
    g.M = B * T; g.N = 8 * kEncH; g.C = w.gin; g.ldc = 8 * kEncH; g.bias = m->enc_lstm_b;
    T2_TRY(gemm_f32(g, s));
  } else {
    // tensor-core path: planes -> 3 x (conv k5 + folded BN + ReLU) -> LSTM input projection (fp32 rows)
    if (a->embedded) T2_TRY(tc_rows_to_planes(a->embedded, (long)T * kEnc, kEnc, kEnc, conv_len, B, T, w.pl0, s));
    else T2_TRY(tc_embed_to_planes(a->text, m->w[W_EMB], m->cfg.n_symbols, conv_len, B, T, w.pl0, s));
    __half* cur = w.pl0; __half* nxt = w.pl1;
    for (int i = 0; i < 3; ++i) {                                                           // model.py:174-175, 194
      const int wb = W_ENC_CONV0 + 7 * i;
      T2_TRY(tc_fold_bn(m->w[wb + 1], m->w[wb + 2], m->w[wb + 3], m->w[wb + 4], m->w[wb + 5], m->cfg.bn_eps, w.scale, w.shift, kEnc, s));
      TcConvArgs c; memset(&c, 0, sizeof(c));
      c.in = cur; c.cin_pad = kEnc; c.wimg = m->tc_enc_conv[i]; c.taps = kConvK; c.B = B; c.T = T; c.cout = kEnc; c.nt_rows = 128;
      c.scale = w.scale; c.shift = w.shift; c.act = 1; c.out_mode = 0; c.out_planes = nxt; c.row_len = conv_len;
      T2_TRY(tc_conv(c, s));
      __half* tmp = cur; cur = nxt; nxt = tmp;
    }
    T2_TRY(tc_fold_bn(m->enc_lstm_b, nullptr, nullptr, nullptr, nullptr, 0.f, w.scale, w.shift, 8 * kEncH, s));
    TcConvArgs c; memset(&c, 0, sizeof(c));
    c.in = cur; c.cin_pad = kEnc; c.wimg = m->tc_enc_wih; c.taps = 1; c.B = B; c.T = T; c.cout = 8 * kEncH; c.nt_rows = 128;
    c.scale = w.scale; c.shift = w.shift; c.act = 0; c.out_mode = 1; c.out_f32 = w.gin; c.ldo = 8 * kEncH;
    T2_TRY(tc_conv(c, s));
  }
  float* hin = w.h; float* hout = w.h + (size_t)2 * B * kEncH;
  T2_CUDA(cudaMemsetAsync(hin, 0, (size_t)2 * B * kEncH * 4, s));
  T2_CUDA(cudaMemsetAsync(w.c, 0, (size_t)2 * B * kEncH * 4, s));
  if (persistent) {
    // persistent recurrence: one cooperative launch for all T steps of both directions
    T2_CUDA(cudaMemsetAsync(hout, 0, (size_t)2 * B * kEncH * 4, s));
    T2_CUDA(cudaMemsetAsync(w.lctrl, 0, sizeof(EncLstmCtrl), s));
    float* hb = w.h;
    const size_t psm = (size_t)(kEncH * 16 + kEncH * 64) * sizeof(float);
    T2_CUDA(cudaFuncSetAttribute(enc_lstm_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psm));
    const float* whf = m->w[W_ENC_LSTM + 1]; const float* whr = m->w[W_ENC_LSTM + 5];
    const int32_t* lens = a->lengths; float* mem = a->memory; int Bv = B, Tv = T;
    void* args[] = {(void*)&w.gin, (void*)&whf, (void*)&whr, (void*)&hb, (void*)&mem, (void*)&lens, (void*)&Bv, (void*)&Tv, (void*)&w.lctrl,
                    (void*)&st_gates, (void*)&st_c};
    T2_CUDA(cudaLaunchCooperativeKernel((void*)enc_lstm_persistent_kernel, dim3(128), dim3(256), args, psm, s));
    g_launch_count++;
    if (a->stash) T2_TRY(encoder_stash_output(a, s));
    return T2_OK;
  }
  const size_t smem = (64 * kEncH + 64 * (kEncH + 1)) * sizeof(float);
  T2_CUDA(cudaFuncSetAttribute(enc_lstm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  for (int step = 0; step < T; ++step) {
    enc_lstm_step_kernel<<<dim3(16, 2, (B + 63) / 64), 256, smem, s>>>(
        w.gin, m->w[W_ENC_LSTM + 1], m->w[W_ENC_LSTM + 5], hin, hout, w.c, a->memory, a->lengths, B, T, step);
    T2_LAUNCH_CHECK();
    float* tmp = hin; hin = hout; hout = tmp;
  }
  return T2_OK;
}

struct PostnetWs {
  float *scale, *shift;    // (512) folded BatchNorm
  __half *pl0, *pl1;       // tensor-core activation planes
  void* train;             // the training conv stack without a stash (on the planes' bytes)
};
static void postnet_ws_layout(Carve& c, int B, int T, PostnetWs* w) {
  w->scale = c.take<float>(kPost); w->shift = c.take<float>(kPost);
  Carve planes = c;
  w->pl0 = planes.take<__half>(tc_planes_bytes(B, T, kPost) / sizeof(__half));
  w->pl1 = planes.take<__half>(tc_planes_bytes(B, T, kPost) / sizeof(__half));
  w->train = c.take<char>(postnet_forward_train_ws_bytes(B, T));
  if (planes.off > c.off) c.off = planes.off;
}
size_t postnet_ws_bytes(int B, int T) { Carve c(nullptr); PostnetWs w; postnet_ws_layout(c, B, T, &w); return c.bytes(); }

// per_row (t2_postnet_infer): every layer's output at t >= lengths[b] is zero too, so row b gets the zero padding each
// convolution sees when the row is its first lengths[b] frames alone.  Otherwise only the input and the output are
// masked and the hidden layers run over the zero frames.
int postnet_forward(T2Model* m, const T2PostnetArgs* a, cudaStream_t s, bool per_row) {
  const int B = a->B, T = a->T;
  const int32_t* layer_len = per_row ? a->lengths : nullptr;
  if (B <= 0 || T <= 0) return fail(T2_ERR_INVALID, "postnet: empty batch");
  if (a->ws_bytes < postnet_ws_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "postnet workspace too small");
  Carve cv(a->ws);
  PostnetWs w;
  postnet_ws_layout(cv, B, T, &w);
  if (a->training || a->stash) return postnet_forward_train(m, a, w.train, s);
  // tensor-core path (model.py:141-146 + residual :511/:524): mel -> planes -> 4 x (conv+BN+tanh) -> conv+BN (+mel)
  const long bs = a->mel_batch_stride ? a->mel_batch_stride : (long)T * kMel;
  T2_TRY(tc_rows_to_planes(a->mel, bs, kMel, 128, a->lengths, B, T, w.pl0, s));
  __half* cur = w.pl0; __half* nxt = w.pl1;
  for (int i = 0; i < 5; ++i) {
    const int wb = W_POST_CONV0 + 7 * i;
    const int cout = i == 4 ? kMel : kPost;
    T2_TRY(tc_fold_bn(m->w[wb + 1], m->w[wb + 2], m->w[wb + 3], m->w[wb + 4], m->w[wb + 5], m->cfg.bn_eps, w.scale, w.shift, cout, s));
    TcConvArgs c; memset(&c, 0, sizeof(c));
    c.in = cur; c.cin_pad = i == 0 ? 128 : kPost; c.wimg = m->tc_post_conv[i]; c.taps = kConvK; c.B = B; c.T = T;
    c.cout = cout; c.nt_rows = i == 4 ? 80 : 128; c.scale = w.scale; c.shift = w.shift; c.act = i == 4 ? 0 : 2;
    if (i < 4) { c.out_mode = 0; c.out_planes = nxt; c.row_len = layer_len; }
    else { c.out_mode = 2; c.out_f32 = a->mel_post; c.residual = a->add_residual ? a->mel : nullptr; c.res_batch_stride = bs; c.row_len = a->lengths; }
    T2_TRY(tc_conv(c, s));
    __half* tmp = cur; cur = nxt; nxt = tmp;
  }
  return T2_OK;
}

}  // namespace t2
