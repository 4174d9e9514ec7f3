// Training path of the Encoder (model.py:173-190) and the Postnet (model.py:141-146): the conv stacks of every
// training-mode forward and every forward under autograd (with a stash for the backward pass or without one), and the
// hand-derived backward.  fp32.
//
// Conv stacks: activations live in a "padded rows" layout -- sequence b occupies rows [b (T+4) + 2, b (T+4) + 2 + T)
// of a (B (T+4), C) channels-last matrix, the 2 rows either side are zero -- so the k=5 convolution is the sum of 5
// plain GEMMs on row-shifted views of the same buffer (no im2col): forward z = sum_k X[r+k-2] W_k^T, input
// gradient g_x = sum_k G_z[r+2-k] W_k, weight gradient dW_k = G_z^T X[r+k-2].  The forward runs these products on the
// tensor-core GEMM (gemm_tc.cu), the input gradient on the implicit-GEMM conv engine (conv_tc.cu) and the weight gradient
// on the wgmma wgrad engine (wgrad_tc.cu); BatchNorm statistics / normalisation / activation / dropout and their backward
// are our kernels.
// BiLSTM backward: reverse recurrence with one skinny GEMM + one elementwise kernel per step and direction.
#include <string.h>

#include <algorithm>

#include "conv_tc.h"
#include "decoder.h"
#include "gemm_f32.cuh"
#include "gemm_tc.h"
#include "train_layers.h"
#include "wgrad_tc.h"

namespace t2 {

namespace {

constexpr int kPadRows = 2;
inline long prow(int b, int t, int T) { return (long)b * (T + 2 * kPadRows) + kPadRows + t; }
__device__ __forceinline__ long d_prow(int b, int t, int T) { return (long)b * (T + 2 * kPadRows) + kPadRows + t; }
// M of the forward conv GEMMs: the padded rows from the first valid row to the last
inline int conv_fwd_rows(int B, int T) { return B * (T + 2 * kPadRows) - 2 * kPadRows; }

// ---- layout conversion ---------------------------------------------------------------------------
// rows (B, T, C) with batch stride -> padded rows (valid rows only; the buffer was zeroed).  len (B) or null: frames
// t >= len[b] count as zero
__global__ void rows_to_padded_kernel(const float* __restrict__ x, long batch_stride, const int32_t* __restrict__ len,
                                      float* __restrict__ xp, int B, int T, int C) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  xp[d_prow(b, t, T) * C + c] = (len == nullptr || t < len[b]) ? x[(long)b * batch_stride + (long)t * C + c] : 0.f;
}
__global__ void embed_to_padded_kernel(const int64_t* __restrict__ text, const float* __restrict__ emb, float* __restrict__ xp,
                                       int B, int T, int n_symbols) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * kEnc) return;
  const int c = (int)(i % kEnc); const long r = i / kEnc; const int t = (int)(r % T); const int b = (int)(r / T);
  long sym = text[r];
  sym = sym < 0 ? 0 : (sym >= n_symbols ? n_symbols - 1 : sym);
  xp[d_prow(b, t, T) * kEnc + c] = emb[sym * kEnc + c];
}

// ---- BatchNorm statistics over the valid rows (training) or running statistics (eval) ----------------
// stats[0..C) = mean of z (without the conv bias), stats[C..2C) = 1/sqrt(var + eps).
// Column reductions run as (C / 32) x kRedSplit blocks writing partial sums, then a small finalize kernel.
constexpr int kRedSplit = 64;
// mode 0: sum z ; mode 1: sum (z - mean)^2 with mean = stats[c]
__global__ void __launch_bounds__(256) bn_partial_kernel(const float* __restrict__ z, int B, int T, int C, int mode,
                                                         const float* __restrict__ stats, float* __restrict__ partial) {
  __shared__ float red[8][33];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const long M = (long)B * T;
  const long per = (M + kRedSplit - 1) / kRedSplit;
  const long r0 = blockIdx.y * per, r1 = r0 + per < M ? r0 + per : M;
  float s = 0.f;
  if (c < C) {
    const float mean = mode ? stats[c] : 0.f;
    for (long r = r0 + rg; r < r1; r += 8) {
      const int b = (int)(r / T), t = (int)(r % T);
      const float d = z[d_prow(b, t, T) * C + c] - mean;
      s += mode ? d * d : d;
    }
  }
  red[rg][cl] = s;
  __syncthreads();
  if (rg == 0 && c < C) {
    float a = 0.f;
    for (int i = 0; i < 8; ++i) a += red[i][cl];
    partial[(long)blockIdx.y * C + c] = a;
  }
}
// mode 0: mean ; mode 1: rstd (+ running statistics) ; mode 2: eval (running statistics -> stats)
__global__ void bn_finalize_kernel(const float* __restrict__ partial, int C, long M, float eps, const float* __restrict__ cbias,
                                   float* run_mean, float* run_var, int mode, float* __restrict__ stats) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (mode == 2) { stats[c] = run_mean[c] - cbias[c]; stats[C + c] = 1.f / sqrtf(run_var[c] + eps); return; }
  double a = 0.0;
  for (int i = 0; i < kRedSplit; ++i) a += (double)partial[(long)i * C + c];
  if (mode == 0) { stats[c] = (float)(a / (double)M); return; }
  const float var = (float)(a / (double)M);
  stats[C + c] = 1.f / sqrtf(var + eps);
  if (run_mean) {   // nn.BatchNorm1d: momentum 0.1, unbiased variance
    run_mean[c] = 0.9f * run_mean[c] + 0.1f * (stats[c] + cbias[c]);
    run_var[c] = 0.9f * run_var[c] + 0.1f * var * ((float)M / (float)(M > 1 ? M - 1 : 1));
  }
}

__device__ __forceinline__ bool conv_keep(const uint8_t* keep, uint64_t seed, uint32_t site, int b, int t, int c, int C, int T) {
  if (keep) return keep[((long)b * C + c) * T + t] != 0;                    // reference layout (B, C, T)
  return philox_keep(seed, site, (uint64_t)((long)b * T + t) * C + c, 0.5f);
}

// y = dropout(act(gamma * xhat + beta)) for the valid rows -> padded rows of the next layer (+ optional plain copy)
__global__ void bn_act_kernel(const float* __restrict__ z, const float* __restrict__ stats, const float* __restrict__ gamma,
                              const float* __restrict__ beta, int B, int T, int C, int act, int dropout, const uint8_t* keep,
                              uint64_t seed, uint32_t site, float* __restrict__ yp, float* __restrict__ y_plain) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  const long pr = d_prow(b, t, T);
  float v = (z[pr * C + c] - stats[c]) * stats[C + c] * gamma[c] + beta[c];
  if (act == ACT_RELU) v = fmaxf(v, 0.f);
  else if (act == ACT_TANH) v = tanhf(v);
  if (dropout) v = conv_keep(keep, seed, site, b, t, c, C, T) ? 2.f * v : 0.f;
  if (yp) yp[pr * C + c] = v;
  if (y_plain) y_plain[i] = v;
}

// backward of bn_act, pass 1: per channel s1 = sum g_ybn, s2 = sum g_ybn * xhat  (g_ybn = gradient wrt gamma*xhat+beta)
// g: gradient wrt the layer output, padded rows (g_padded) or plain (B*T, C) rows.
__device__ __forceinline__ float g_ybn_at(const float* g, int g_padded, const float* y, int b, int t, int c, int C, int T, int act,
                                          int dropout, const uint8_t* keep, uint64_t seed, uint32_t site) {
  const long pr = d_prow(b, t, T);
  float gv = g[(g_padded ? pr : ((long)b * T + t)) * C + c];
  float a = y[pr * C + c];
  if (dropout) {
    if (!conv_keep(keep, seed, site, b, t, c, C, T)) return 0.f;
    gv *= 2.f; a *= 0.5f;
  }
  if (act == ACT_RELU) return a > 0.f ? gv : 0.f;
  if (act == ACT_TANH) return gv * (1.f - a * a);
  return gv;
}
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const float* __restrict__ g, int g_padded, const float* __restrict__ y,
                                                            const float* __restrict__ z, const float* __restrict__ stats, int B, int T,
                                                            int C, int act, int dropout, const uint8_t* keep, uint64_t seed,
                                                            uint32_t site, float* __restrict__ partial) {
  __shared__ float r1[8][33], r2[8][33];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const long M = (long)B * T;
  const long per = (M + kRedSplit - 1) / kRedSplit;
  const long q0 = blockIdx.y * per, q1 = q0 + per < M ? q0 + per : M;
  float s1 = 0.f, s2 = 0.f;
  if (c < C) {
    const float mean = stats[c], rstd = stats[C + c];
    for (long r = q0 + rg; r < q1; r += 8) {
      const int b = (int)(r / T), t = (int)(r % T);
      const float gy = g_ybn_at(g, g_padded, y, b, t, c, C, T, act, dropout, keep, seed, site);
      s1 += gy;
      s2 = fmaf(gy, (z[d_prow(b, t, T) * C + c] - mean) * rstd, s2);
    }
  }
  r1[rg][cl] = s1; r2[rg][cl] = s2;
  __syncthreads();
  if (rg == 0 && c < C) {
    float a1 = 0.f, a2 = 0.f;
    for (int i = 0; i < 8; ++i) { a1 += r1[i][cl]; a2 += r2[i][cl]; }
    partial[((long)blockIdx.y * 2 + 0) * C + c] = a1;
    partial[((long)blockIdx.y * 2 + 1) * C + c] = a2;
  }
}
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ partial, int C, float* __restrict__ sums) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;     // sums[0..C) = d beta, sums[C..2C) = d gamma
  if (i >= 2 * C) return;
  const int which = i / C, c = i - which * C;
  double a = 0.0;
  for (int k = 0; k < kRedSplit; ++k) a += (double)partial[((long)k * 2 + which) * C + c];
  sums[i] = (float)a;
}
// pass 2: g_z = gamma rstd (g_ybn - s1/M - xhat s2/M)  (training)  |  gamma rstd g_ybn  (eval), valid rows of a zeroed buffer
__global__ void bn_bwd_apply_kernel(const float* __restrict__ g, int g_padded, const float* __restrict__ y, const float* __restrict__ z,
                                    const float* __restrict__ stats, const float* __restrict__ gamma, const float* __restrict__ sums,
                                    int B, int T, int C, int act, int dropout, int training, const uint8_t* keep, uint64_t seed,
                                    uint32_t site, float* __restrict__ gz) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  const long pr = d_prow(b, t, T);
  const float gy = g_ybn_at(g, g_padded, y, b, t, c, C, T, act, dropout, keep, seed, site);
  const float rstd = stats[C + c];
  float v = gy;
  if (training) {
    const float xhat = (z[pr * C + c] - stats[c]) * rstd;
    const float inv_m = 1.f / (float)((long)B * T);
    v = gy - sums[c] * inv_m - xhat * sums[C + c] * inv_m;
  }
  gz[pr * C + c] = v * gamma[c] * rstd;
}
// zero the rows t >= len[b] of a padded-rows buffer
__global__ void mask_padded_rows_kernel(float* __restrict__ xp, const int32_t* __restrict__ len, int B, int T, int C) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  if (t >= len[b]) xp[d_prow(b, t, T) * C + c] = 0.f;
}
__global__ void fill1_kernel(float* p, float v, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
// padded rows (valid) -> (B, C, T) with optional residual; len (B) or null: zero at t >= len[b]
__global__ void rows_to_bct_kernel(const float* __restrict__ yp, const float* __restrict__ res_p, const int32_t* __restrict__ len,
                                   float* __restrict__ out, int B, int T, int C) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int t = (int)(i % T); const long r = i / T; const int c = (int)(r % C); const int b = (int)(r / C);
  const long pr = d_prow(b, t, T);
  float v = yp[pr * C + c];
  if (res_p) v += res_p[pr * C + c];
  if (len && t >= len[b]) v = 0.f;
  out[i] = v;
}
// gradient (B, C, T) -> plain rows (B*T, C)
__global__ void bct_to_rows_kernel(const float* __restrict__ g, float* __restrict__ rows, int B, int T, int C) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  rows[i] = g[((long)b * C + c) * T + t];
}
// d_x rows (B, T, C) = padded gradient (valid rows) [+ plain rows]
__global__ void padded_to_rows_kernel(const float* __restrict__ gp, const float* __restrict__ add_rows, float* __restrict__ out,
                                      int B, int T, int C) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * C) return;
  const int c = (int)(i % C); const long r = i / C; const int t = (int)(r % T); const int b = (int)(r / T);
  float v = gp[d_prow(b, t, T) * C + c];
  if (add_rows) v += add_rows[i];
  out[i] = v;
}
// embedding gradient: one block per symbol; the block first lists the positions that hold its symbol (ascending, so the
// summation order is fixed), then adds their gradient rows                                    model.py:503
__global__ void __launch_bounds__(256) embed_bwd_kernel(const int64_t* __restrict__ text, const float* __restrict__ gp,
                                                        float* __restrict__ d_emb, int B, int T, int n_symbols) {
  extern __shared__ int s_rows[];                      // (B * T) matching positions, compacted
  __shared__ int s_cnt[256 + 1];
  const int sym = blockIdx.x, tid = threadIdx.x;
  const int M = B * T;
  const int per = (M + 255) / 256;
  const int r0 = tid * per, r1 = r0 + per < M ? r0 + per : M;
  int cnt = 0;
  for (int r = r0; r < r1; ++r) {
    long v = text[r];
    v = v < 0 ? 0 : (v >= n_symbols ? n_symbols - 1 : v);
    cnt += v == sym;
  }
  s_cnt[tid + 1] = cnt;
  if (tid == 0) s_cnt[0] = 0;
  __syncthreads();
  if (tid == 0) for (int i = 1; i <= 256; ++i) s_cnt[i] += s_cnt[i - 1];
  __syncthreads();
  int o = s_cnt[tid];
  for (int r = r0; r < r1; ++r) {
    long v = text[r];
    v = v < 0 ? 0 : (v >= n_symbols ? n_symbols - 1 : v);
    if (v == sym) s_rows[o++] = r;
  }
  __syncthreads();
  const int n = s_cnt[256];
  for (int c = tid; c < kEnc; c += 256) {
    float s = 0.f;
    for (int i = 0; i < n; ++i) {
      const int r = s_rows[i];
      s += gp[d_prow(r / T, r % T, T) * kEnc + c];
    }
    d_emb[(long)sym * kEnc + c] = s;
  }
}

// ---- one conv + BatchNorm + activation + dropout layer -------------------------------------------------
struct ConvLayer {
  int cin, cout, act, dropout;       // dropout only when the module is in training mode
  const float* wpk;                  // packed fp32 weights (cout, 5, cin)
  int wbase;                         // index of conv.weight in the state_dict table
  uint32_t site; const uint8_t* keep;
};
// The training FORWARD convs stay on 5 row-shifted gemm_tc products (one accumulation chain per 64-wide K chunk, 7e-7):
// the conv engine accumulates ~100-480 MMAs in one chain (3e-6 ... 1e-5 output error; the accumulator update truncates)
// and near-constant BatchNorm channels amplify that to a 2e-2 gradient error on one ill-conditioned test shape.  The
// input gradients run on the conv engine.
// Wd[ci][co][k'] = W[co][ci][4 - k']: the input gradient of a k=5 'same' conv is a conv of G_z with this kernel
__global__ void flip_conv_w_kernel(const float* __restrict__ w, float* __restrict__ wd, int cout, int cin) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)cout * cin * kConvK) return;
  const int k = (int)(i % kConvK); const long r = i / kConvK; const int ci = (int)(r % cin); const int co = (int)(r / cin);
  wd[((long)ci * cout + co) * kConvK + (kConvK - 1 - k)] = w[i];
}
// s_g = the power-of-two scale of the largest channel of G_z: max |G_z| = f 2^e with f in [0.5, 1) gives s_g = 2^-e, with
// the clamp of the per-channel scales (wg_colstats_finalize_kernel).  It is read from the column maxima wg_colstats left
// in its partials, so all-zero channels play no part (their own scale is 1, which would win a minimum over the channel
// scales whenever max |G_z| < 0.5 and leave tiny gradients unscaled, in the fp16 subnormal range); s_g = 1 when G_z is
// all zero.  out_vec[0..512) = 1 / s_g.  part and out_vec may alias: every read precedes the first barrier.
__global__ void __launch_bounds__(256) global_scale_kernel(const float* part, int C, float* __restrict__ s_g, float* out_vec) {
  __shared__ float red[256];
  float mx = 0.f;
  for (int i = threadIdx.x; i < kWgStatSplit * C; i += 256) mx = fmaxf(mx, part[(long)(i / C) * 2 * C + i % C]);
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  int e = 0;
  if (red[0] > 0.f && red[0] < 3.0e38f) frexpf(red[0], &e);
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  if (threadIdx.x == 0) *s_g = ldexpf(1.f, -e);
  for (int i = threadIdx.x; i < 512; i += 256) out_vec[i] = ldexpf(1.f, e);
}
int tc_train_conv(T2Model* m, const float* xp, int cin, const uint8_t* wimg, int cout, int B, int T, float* outp, __half* planes,
                  const float* in_scale, const float* out_scale, cudaStream_t s) {
  // outp[padded rows][cout] = conv_k5(xp[padded rows][cin]) (no bias), split-fp16 tensor-core engine; the input is
  // pre-scaled by the device scalar *in_scale (a power of two) and out_scale[c] = 1 / *in_scale undoes it
  const int c_pad = cin < 128 ? 128 : cin;
  T2_TRY(tc_rows_to_planes_scaled(xp + (long)kPadRows * cin, (long)(T + 2 * kPadRows) * cin, cin, c_pad, nullptr, B, T, planes,
                                  in_scale, s));
  TcConvArgs c;
  memset(&c, 0, sizeof(c));
  c.in = planes; c.cin_pad = c_pad; c.wimg = wimg; c.taps = kConvK; c.B = B; c.T = T; c.cout = cout; c.nt_rows = cout >= 128 ? 128 : 80;
  c.scale = out_scale; c.shift = m->zeros; c.act = 0; c.out_mode = 1;
  c.out_f32 = outp + (long)kPadRows * cout; c.ldo = cout; c.out_seq_rows = T + 2 * kPadRows;
  return tc_conv(c, s);
}

// ---- conv weight gradient on the wgmma engine (wgrad_tc.cu) ---------------------------------------------------------
// dW_k[co][ci] = sum_r G_z[r][co] X[r + k - 2][ci]: K = padded rows in chunks of 64, A = G_z^T images (per-channel power-of-two
// scale), B = X^T images, one set per tap (source rows shifted by k - 2), 128 x 256 tiles, K splits reduced in a fixed order.
struct WgConvWs { uint8_t* img_a; uint8_t* img_b; float* part; float* stat; float* scale; float* inv; float* colsum; };
void wgconv_layout(Carve& c, int B, int T, WgConvWs* w) {    // every region 1024-aligned
  const long Mp = (long)B * (T + 2 * kPadRows);
  const long nch = (Mp + 63) / 64;
  const int seg = wgrad_seg((int)nch), nsplit = (int)((nch + seg - 1) / seg);
  w->img_a = c.take<uint8_t>((size_t)nch * 4 * kWgTileA, 1024);                 // cout <= 512: 4 tiles of 128 rows
  w->img_b = c.take<uint8_t>((size_t)kConvK * nch * 2 * kWgTileB, 1024);        // cin <= 512: 2 tiles of 256 rows, 5 taps
  w->part = c.take<float>((size_t)nsplit * 512 * (kConvK * 512), 1024);
  w->stat = c.take<float>(wg_colstats_ws_bytes(512) / sizeof(float), 1024);
  w->scale = c.take<float>(512, 1024); w->inv = c.take<float>(512, 1024); w->colsum = c.take<float>(512, 1024);
}
__global__ void wgconv_reduce_kernel(const float* __restrict__ part, int nsplit, int coutP, int ldp, int cinP, int cout, int cin,
                                     float* __restrict__ dW) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;       // dW (co, ci, k) state_dict layout
  if (i >= (long)cout * cin * kConvK) return;
  const int k = (int)(i % kConvK); const long r = i / kConvK; const int ci = (int)(r % cin); const int co = (int)(r / cin);
  float s = 0.f;
  for (int sp = 0; sp < nsplit; ++sp) s += part[((long)sp * coutP + co) * ldp + (long)k * cinP + ci];
  dW[i] = s;
}
int conv_wgrad_tc(const ConvLayer& L, int B, int T, const float* gz_p, const float* xp, float* dW, float* d_cbias, const WgConvWs& w,
                  cudaStream_t s) {
  const long Mp = (long)B * (T + 2 * kPadRows);
  const int nch = (int)((Mp + 63) / 64);
  const int seg = wgrad_seg(nch), nsplit = (nch + seg - 1) / seg;
  const int ntA = (L.cout + 127) / 128, ntB = (L.cin + 255) / 256;
  const int coutP = ntA * 128, cinP = ntB * 256, ldp = kConvK * cinP;
  fill1_kernel<<<2, 256, 0, s>>>(w.inv, 1.f, 512);
  T2_LAUNCH_CHECK();
  T2_TRY(wg_colstats(gz_p, Mp, L.cout, w.stat, w.scale, w.inv, w.colsum, s));
  if (d_cbias) T2_CUDA(cudaMemcpyAsync(d_cbias, w.colsum, (size_t)L.cout * 4, cudaMemcpyDeviceToDevice, s));
  if (!dW) return T2_OK;
  T2_TRY(wg_transpose_images(gz_p, L.cout, 0, Mp, 64, nch, L.cout, 128, w.scale, w.img_a, s));
  const size_t b_img = (size_t)nch * ntB * kWgTileB;
  for (int k = 0; k < kConvK; ++k)
    T2_TRY(wg_transpose_images(xp, L.cin, k - kPadRows, Mp, 64, nch, L.cin, 256, nullptr, w.img_b + (size_t)k * b_img, s));
  const WgConvJobs jobs = {w.img_a, w.img_b, b_img, w.part, w.inv, nch, seg, nsplit, ntA, ntB, coutP, cinP, ldp};
  T2_TRY(wg_run_jobs(jobs, s));
  const long n = (long)L.cout * L.cin * kConvK;
  wgconv_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.part, nsplit, coutP, ldp, cinP, L.cout, L.cin, dW);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

// gemm / gemm_bytes: the scratch of the forward GEMMs (stack_ws_layout)
int conv_fwd(T2Model* m, const ConvLayer& L, int B, int T, int training, uint64_t seed, const float* xp, float* zp,
             float* stats, float* yp, float* y_plain, bool update_running, float* partial, void* gemm, size_t gemm_bytes,
             cudaStream_t s) {
  const int Me = conv_fwd_rows(B, T);
  for (int k = 0; k < kConvK; ++k)
    T2_TRY(gemm_tc_rm(m->sm_count, s, gemm, gemm_bytes, false, true, Me, L.cout, L.cin, xp + (long)k * L.cin, L.cin,
                      L.wpk + (long)k * L.cin, (long)kConvK * L.cin, zp + (long)kPadRows * L.cout, L.cout, k ? 1.f : 0.f));
  {
    float* rm = const_cast<float*>(m->w[L.wbase + 4]); float* rv = const_cast<float*>(m->w[L.wbase + 5]);
    const long M = (long)B * T;
    if (!training) {
      bn_finalize_kernel<<<(L.cout + 127) / 128, 128, 0, s>>>(nullptr, L.cout, M, m->cfg.bn_eps, m->w[L.wbase + 1], rm, rv, 2, stats);
      T2_LAUNCH_CHECK();
    } else {
      for (int mode = 0; mode < 2; ++mode) {
        bn_partial_kernel<<<dim3((L.cout + 31) / 32, kRedSplit), 256, 0, s>>>(zp, B, T, L.cout, mode, stats, partial);
        T2_LAUNCH_CHECK();
        bn_finalize_kernel<<<(L.cout + 127) / 128, 128, 0, s>>>(partial, L.cout, M, m->cfg.bn_eps, m->w[L.wbase + 1],
                                                                update_running ? rm : nullptr, rv, mode, stats);
        T2_LAUNCH_CHECK();
      }
    }
  }
  const long n = (long)B * T * L.cout;
  bn_act_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(zp, stats, m->w[L.wbase + 2], m->w[L.wbase + 3], B, T, L.cout, L.act,
                                                             L.dropout, L.keep, seed, L.site, yp, y_plain);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

// The scratch of conv_bwd, shared by the layers of a stack in stream order.  Every layer of either stack has at most 512
// input and 512 output channels.
struct ConvBwdWs {
  WgConvWs wg;
  __half* planes;          // input planes of the input-gradient conv
  float* wflip;            // (512, 512, 5) the flipped / transposed weights of the input-gradient conv
  uint8_t* wimg;           // their packed image
};
void conv_bwd_layout(Carve& c, int B, int T, ConvBwdWs* w) {
  wgconv_layout(c, B, T, &w->wg);
  w->planes = c.take<__half>(tc_planes_bytes(B, T, 512) / sizeof(__half));
  w->wflip = c.take<float>((size_t)512 * 512 * kConvK);
  w->wimg = c.take<uint8_t>(tc_weights_bytes(512, 512, kConvK, 128), 1024);
}

// g: gradient wrt the layer output (padded or plain rows).  Writes gx_p (padded rows, garbage in the pad rows) when
// non-null, and the gradients of conv.weight / conv.bias / bn.weight / bn.bias.
int conv_bwd(T2Model* m, const ConvLayer& L, int B, int T, int training, uint64_t seed, const float* g, int g_padded,
             const float* xp, const float* zp, const float* stats, const float* yp, float* gz_p, float* gx_p, float* sums,
             float* const* G, const ConvBwdWs& cw, cudaStream_t s) {
  const WgConvWs& wg = cw.wg;
  const long Mp = (long)B * (T + 2 * kPadRows);
  float* partial = sums + 2 * L.cout;      // (kRedSplit, 2, cout) scratch behind the two result rows
  bn_bwd_reduce_kernel<<<dim3((L.cout + 31) / 32, kRedSplit), 256, 0, s>>>(g, g_padded, yp, zp, stats, B, T, L.cout, L.act, L.dropout,
                                                                            L.keep, seed, L.site, partial);
  T2_LAUNCH_CHECK();
  bn_bwd_finalize_kernel<<<(2 * L.cout + 127) / 128, 128, 0, s>>>(partial, L.cout, sums);
  T2_LAUNCH_CHECK();
  T2_CUDA(cudaMemsetAsync(gz_p, 0, (size_t)Mp * L.cout * 4, s));
  const long n = (long)B * T * L.cout;
  bn_bwd_apply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(g, g_padded, yp, zp, stats, m->w[L.wbase + 2], sums, B, T, L.cout, L.act,
                                                                   L.dropout, training, L.keep, seed, L.site, gz_p);
  T2_LAUNCH_CHECK();
  if (G[L.wbase + 3]) T2_CUDA(cudaMemcpyAsync(G[L.wbase + 3], sums, (size_t)L.cout * 4, cudaMemcpyDeviceToDevice, s));           // d beta
  if (G[L.wbase + 2]) T2_CUDA(cudaMemcpyAsync(G[L.wbase + 2], sums + L.cout, (size_t)L.cout * 4, cudaMemcpyDeviceToDevice, s));  // d gamma
  // weight + bias gradient on our wgmma engine
  T2_TRY(conv_wgrad_tc(L, B, T, gz_p, xp, G[L.wbase], G[L.wbase + 1], wg, s));
  if (gx_p) {   // input gradient = conv of G_z with the flipped / transposed kernel on the tensor-core engine
    // G_z is pre-scaled by a power of two (from the per-channel statistics of the weight-gradient pass): fp16 range
    global_scale_kernel<<<1, 256, 0, s>>>(wg.stat, L.cout, wg.colsum, wg.stat);       // colsum[0] = s_g, stat[0..512) = 1 / s_g
    T2_LAUNCH_CHECK();
    const long nw = (long)L.cout * L.cin * kConvK;
    flip_conv_w_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(m->w[L.wbase], cw.wflip, L.cout, L.cin);
    T2_LAUNCH_CHECK();
    T2_TRY(tc_pack_weights(cw.wflip, L.cin, L.cout, kConvK, L.cin >= 128 ? 128 : 80, cw.wimg, s));
    T2_TRY(tc_train_conv(m, gz_p, L.cout, cw.wimg, L.cin, B, T, gx_p, cw.planes, wg.colsum, wg.stat, s));
  }
  return T2_OK;
}

// ---- stash layouts ---------------------------------------------------------------------------------
struct StackStash {        // L conv layers: X_0..X_L (padded), Z_0..Z_{L-1} (padded), stats (2 C each)
  float* x[6]; float* z[5]; float* stats[5];
};
void stack_layout(Carve& c, int B, int T, int L, const int* ch, StackStash* st) {
  const size_t Mp = (size_t)B * (T + 2 * kPadRows);
  memset(st, 0, sizeof(*st));
  for (int l = 0; l <= L; ++l) st->x[l] = c.take<float>(Mp * ch[l]);
  for (int l = 0; l < L; ++l) st->z[l] = c.take<float>(Mp * ch[l + 1]);
  for (int l = 0; l < L; ++l) st->stats[l] = c.take<float>((size_t)(2 + kRedSplit) * ch[l + 1]);   // + reduction scratch
}
// The same stack without a stash (a training-mode forward outside autograd), laid out on the caller's workspace.  Nothing
// is kept for a backward pass: two padded buffers take turns as the layers' inputs and outputs, and one z / statistics
// region serves every layer.  keep_input: the input gets a buffer of its own (the postnet adds it back as the residual).
// The activation buffers come first, then z and the statistics, and last the scratch of the forward GEMMs, which a
// forward with a stash uses too.
void stack_ws_layout(Carve& c, int B, int T, int L, const int* ch, bool keep_input, StackStash* st, void** gemm,
                     size_t* gemm_bytes) {
  const size_t Mp = (size_t)B * (T + 2 * kPadRows);
  int cmax = 0;
  *gemm_bytes = 0;
  for (int l = 0; l <= L; ++l) cmax = ch[l] > cmax ? ch[l] : cmax;
  for (int l = 0; l < L; ++l) *gemm_bytes = std::max(*gemm_bytes, gemm_tc_ws_bytes(conv_fwd_rows(B, T), ch[l + 1], ch[l]));
  memset(st, 0, sizeof(*st));
  float* in = keep_input ? c.take<float>(Mp * ch[0]) : nullptr;
  float* buf[2] = {c.take<float>(Mp * cmax), c.take<float>(Mp * cmax)};
  for (int l = 0; l <= L; ++l) st->x[l] = (l == 0 && in) ? in : buf[l & 1];
  float* z = c.take<float>(Mp * cmax);
  float* stats = c.take<float>((size_t)(2 + kRedSplit) * cmax);
  for (int l = 0; l < L; ++l) { st->z[l] = z; st->stats[l] = stats; }
  *gemm = c.take<char>(*gemm_bytes);
}
const int kPostCh[6] = {kMel, kPost, kPost, kPost, kPost, kMel};
const int kEncCh[4] = {kEnc, kEnc, kEnc, kEnc};

struct EncStash {
  StackStash cs;
  float* xl;       // (B*T, 512) conv stack output (plain rows) = LSTM input
  float* gates;    // (B, T, 2048) LSTM gate activations, forward | reverse, i f g o
  float* cst;      // (B, T, 512) cell states
  float* mem;      // (B, T, 512) copy of the output (h of every valid step)
};
void enc_stash_layout(Carve& c, int B, int T, EncStash* st) {
  stack_layout(c, B, T, 3, kEncCh, &st->cs);
  st->xl = c.take<float>((size_t)B * T * kEnc);
  st->gates = c.take<float>((size_t)B * T * 8 * kEncH);
  st->cst = c.take<float>((size_t)B * T * kEnc); st->mem = c.take<float>((size_t)B * T * kEnc);
}
// the stash of a forward call, laid out on the caller's buffer
EncStash enc_stash(const void* stash, int B, int T) {
  Carve c(const_cast<void*>(stash));
  EncStash st;
  enc_stash_layout(c, B, T, &st);
  return st;
}

// ---- encoder LSTM backward ------------------------------------------------------------------------------
// elementwise part of one reverse step of both directions.  grid (2, B), block 256 = hidden units.
__global__ void __launch_bounds__(256) enc_lstm_bwd_kernel(const float* __restrict__ d_mem, const float* __restrict__ part, int has_part,
                                                           const float* __restrict__ gates, const float* __restrict__ cst,
                                                           const int32_t* __restrict__ lengths, float* __restrict__ g_c,
                                                           float* __restrict__ dG, int B, int T, int step, int nsplit) {
  const int dir = blockIdx.x, b = blockIdx.y, u = threadIdx.x;
  const int t = dir == 0 ? T - 1 - step : step;          // backward order of each direction
  const bool valid = lengths == nullptr || t < lengths[b];
  float* dg = dG + (((long)b * T + t) * 2 + dir) * (4 * kEncH) + u;
  const long ci = ((long)dir * B + b) * kEncH + u;
  if (!valid) {
    dg[0] = 0.f; dg[kEncH] = 0.f; dg[2 * kEncH] = 0.f; dg[3 * kEncH] = 0.f;
    g_c[ci] = 0.f;
    return;
  }
  float g_h = d_mem[((long)b * T + t) * kEnc + dir * kEncH + u];
  if (has_part)
    for (int s = 0; s < nsplit; ++s) g_h += part[(((long)dir * nsplit + s) * 64 + b) * kEncH + u];
  const float* gp = gates + ((long)b * T + t) * (8 * kEncH) + dir * 4 * kEncH + u;
  const float gi = gp[0], gf = gp[kEncH], gg = gp[2 * kEncH], go = gp[3 * kEncH];
  const int tp = dir == 0 ? t - 1 : t + 1;               // previous step of the forward recurrence
  const float c = cst[((long)b * T + t) * kEnc + dir * kEncH + u];
  const float cp = (tp >= 0 && tp < T) ? cst[((long)b * T + tp) * kEnc + dir * kEncH + u] : 0.f;
  const float tc = tanhf(c);
  const float d_o = g_h * tc;
  const float d_c = g_c[ci] + g_h * go * (1.f - tc * tc);
  dg[0] = d_c * gg * gi * (1.f - gi);
  dg[kEncH] = d_c * cp * gf * (1.f - gf);
  dg[2 * kEncH] = d_c * gi * (1.f - gg * gg);
  dg[3 * kEncH] = d_o * go * (1.f - go);
  g_c[ci] = d_c * gf;
}
// g_h' partials = dG_t (B x 1024) . W_hh (1024 x 256) per direction.  grid (2 column tiles, nsplit, 2 dirs), 64 x 128 tiles
__global__ void __launch_bounds__(256) enc_whh_bwd_kernel(const float* __restrict__ dG, const float* __restrict__ whh_f,
                                                          const float* __restrict__ whh_r, float* __restrict__ part, int B, int T,
                                                          int step, int nsplit) {
  constexpr int BK = 32;
  __shared__ __align__(16) float As[BK][64 + 4];
  __shared__ __align__(16) float Bs[BK][128];
  const int dir = blockIdx.z, tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const int t = dir == 0 ? T - 1 - step : step;
  const float* W = (dir == 0 ? whh_f : whh_r) + blockIdx.x * 128;
  const int per = 4 * kEncH / nsplit;
  const int n_begin = blockIdx.y * per, n_end = n_begin + per;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int n0 = n_begin; n0 < n_end; n0 += BK) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int idx = tid * 2 + i, r = idx >> 3, q = idx & 7;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < B) v = *reinterpret_cast<const float4*>(dG + (((long)r * T + t) * 2 + dir) * (4 * kEncH) + n0 + q * 4);
      As[q * 4 + 0][r] = v.x; As[q * 4 + 1][r] = v.y; As[q * 4 + 2][r] = v.z; As[q * 4 + 3][r] = v.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * 256, kk = idx >> 5, c4 = idx & 31;
      *reinterpret_cast<float4*>(&Bs[kk][c4 * 4]) = __ldg(reinterpret_cast<const float4*>(W + (long)(n0 + kk) * kEncH + c4 * 4));
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
  float* out = part + (((long)dir * nsplit + blockIdx.y) * 64 + ty * 8) * kEncH + blockIdx.x * 128 + tx * 4;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    *reinterpret_cast<float4*>(out + (long)i * kEncH) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}
// h of the previous forward-recurrence step of every (b, t, dir): rows for the W_hh gradient GEMM
__global__ void enc_hprev_kernel(const float* __restrict__ mem, float* __restrict__ hp, int B, int T) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T * kEnc) return;
  const int c = (int)(i % kEnc); const long r = i / kEnc; const int t = (int)(r % T); const int b = (int)(r / T);
  const int dir = c / kEncH;
  const int tp = dir == 0 ? t - 1 : t + 1;
  hp[i] = (tp >= 0 && tp < T) ? mem[((long)b * T + tp) * kEnc + c] : 0.f;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// Postnet
// ---------------------------------------------------------------------------------------------------
size_t postnet_stash_bytes(int B, int T) { Carve c(nullptr); StackStash st; stack_layout(c, B, T, 5, kPostCh, &st); return c.bytes(); }
size_t postnet_forward_train_ws_bytes(int B, int T) {
  Carve c(nullptr);
  StackStash st;
  void* gemm; size_t gemm_bytes;
  stack_ws_layout(c, B, T, 5, kPostCh, true, &st, &gemm, &gemm_bytes);
  return c.bytes();
}

static void post_layers(T2Model* m, int training, const uint8_t* keep, int B, int T, ConvLayer* L) {
  for (int i = 0; i < 5; ++i) {
    L[i].cin = kPostCh[i]; L[i].cout = kPostCh[i + 1]; L[i].act = i == 4 ? ACT_NONE : ACT_TANH; L[i].dropout = training;
    L[i].wpk = m->post_conv_w[i]; L[i].wbase = W_POST_CONV0 + 7 * i; L[i].site = 2000 + i;
    L[i].keep = (training && keep) ? keep + (size_t)i * B * kPost * T : nullptr;     // [(B,512,T)] x 4 + (B,80,T)
  }
}

int postnet_forward_train(T2Model* m, const T2PostnetArgs* a, void* ws, cudaStream_t s) {
  const int B = a->B, T = a->T;
  if (a->stash && a->lengths) return fail(T2_ERR_UNSUPPORTED, "postnet: the training stash path takes no length mask (model.py:510)");
  if (a->stash && a->stash_bytes < postnet_stash_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "postnet stash too small");
  StackStash st;
  void* gemm; size_t gemm_bytes;
  Carve wc(ws);
  stack_ws_layout(wc, B, T, 5, kPostCh, true, &st, &gemm, &gemm_bytes);
  if (a->stash) {
    Carve c(a->stash);
    stack_layout(c, B, T, 5, kPostCh, &st);
    T2_CUDA(cudaMemsetAsync(st.x[0], 0, c.off, s));      // zero pad rows everywhere
  } else {
    T2_CUDA(cudaMemsetAsync(st.x[0], 0, (char*)st.z[0] - (char*)st.x[0], s));   // the activations, pad rows included
  }
  const long n = (long)B * T * kMel;
  rows_to_padded_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->mel, a->mel_batch_stride ? a->mel_batch_stride : (long)T * kMel,
                                                                     a->lengths, st.x[0], B, T, kMel);
  T2_LAUNCH_CHECK();
  ConvLayer L[5];
  post_layers(m, a->training, a->keep, B, T, L);
  for (int i = 0; i < 5; ++i)
    T2_TRY(conv_fwd(m, L[i], B, T, a->training, a->seed, st.x[i], st.z[i], st.stats[i], st.x[i + 1], nullptr, a->training != 0,
                    st.stats[i] + 2 * L[i].cout, gemm, gemm_bytes, s));
  rows_to_bct_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st.x[5], a->add_residual ? st.x[0] : nullptr, a->lengths, a->mel_post,
                                                                  B, T, kMel);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

struct PostBwdWs {
  float *gz, *gxa, *gxb;   // padded rows (B (T+4), 512)
  float* grow;             // (B T, 80) output gradient rows
  float* sums;
  ConvBwdWs cw;
};
static void postnet_backward_ws_layout(Carve& c, int B, int T, PostBwdWs* w) {
  const size_t Mp = (size_t)B * (T + 2 * kPadRows);
  w->gz = c.take<float>(Mp * kPost); w->gxa = c.take<float>(Mp * kPost); w->gxb = c.take<float>(Mp * kPost);
  w->grow = c.take<float>((size_t)B * T * kMel);
  w->sums = c.take<float>((size_t)(2 + 2 * kRedSplit) * kPost);
  conv_bwd_layout(c, B, T, &w->cw);
}
size_t postnet_backward_ws_bytes(int B, int T) {
  Carve c(nullptr, 1024);
  PostBwdWs w;
  postnet_backward_ws_layout(c, B, T, &w);
  return c.bytes();
}

int postnet_backward(T2Model* m, const T2PostnetBwdArgs* a, cudaStream_t s) {
  const int B = a->B, T = a->T;
  if (a->n_grads != W_COUNT) return fail(T2_ERR_INVALID, "postnet backward: expected %d gradient pointers", (int)W_COUNT);
  if (a->ws_bytes < postnet_backward_ws_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "postnet backward workspace too small");
  if (a->stash_bytes < postnet_stash_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "postnet stash too small");
  StackStash st;
  Carve sc(const_cast<void*>(a->stash));
  stack_layout(sc, B, T, 5, kPostCh, &st);
  PostBwdWs w;
  Carve wc(a->ws, 1024);
  postnet_backward_ws_layout(wc, B, T, &w);
  const long n = (long)B * T * kMel;
  bct_to_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->d_mel_post, w.grow, B, T, kMel);     // (B,80,T) -> rows
  T2_LAUNCH_CHECK();
  ConvLayer L[5];
  post_layers(m, a->training, a->keep, B, T, L);
  const float* g = w.grow; int g_padded = 0;
  float* gx = w.gxa;
  for (int i = 4; i >= 0; --i) {
    if (i == 0 && a->wgrad_lengths) {   // the stash is consumed by this call: mask the stored input in place
      mask_padded_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st.x[0], a->wgrad_lengths, B, T, kMel);
      T2_LAUNCH_CHECK();
    }
    T2_TRY(conv_bwd(m, L[i], B, T, a->training, a->seed, g, g_padded, st.x[i], st.z[i], st.stats[i], st.x[i + 1], w.gz, gx, w.sums,
                    a->grads, w.cw, s));
    g = gx; g_padded = 1;
    gx = gx == w.gxa ? w.gxb : w.gxa;
  }
  if (a->d_mel) {   // gradient wrt the postnet input (B, T, 80) (+ the residual branch, model.py:511)
    padded_to_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(g, a->add_residual ? w.grow : nullptr, a->d_mel, B, T, kMel);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

// ---------------------------------------------------------------------------------------------------
// Encoder
// ---------------------------------------------------------------------------------------------------
size_t encoder_stash_bytes(int B, int T) { Carve c(nullptr); EncStash st; enc_stash_layout(c, B, T, &st); return c.bytes(); }

static void enc_layers(T2Model* m, int training, const uint8_t* keep, int B, int T, ConvLayer* L) {
  for (int i = 0; i < 3; ++i) {
    L[i].cin = kEnc; L[i].cout = kEnc; L[i].act = ACT_RELU; L[i].dropout = training;
    L[i].wpk = m->enc_conv_w[i]; L[i].wbase = W_ENC_CONV0 + 7 * i; L[i].site = 1000 + i;
    L[i].keep = (training && keep) ? keep + (size_t)i * B * kEnc * T : nullptr;
  }
}

size_t encoder_convs_train_ws_bytes(int B, int T) {
  Carve c(nullptr);
  StackStash st;
  void* gemm; size_t gemm_bytes;
  stack_ws_layout(c, B, T, 3, kEncCh, false, &st, &gemm, &gemm_bytes);
  return c.bytes();
}

// conv stack of the training forward: returns the LSTM input rows (B*T, 512).  With a stash it fills the stash and
// returns where the BiLSTM keeps its gates / cell states; without one it runs on ws and *gates = *cst = null.  Either way
// the GEMMs take their scratch from ws.
int encoder_convs_train(T2Model* m, const T2EncoderArgs* a, void* ws, cudaStream_t s, const float** xl, float** gates, float** cst) {
  const int B = a->B, T = a->T;
  if (a->stash && a->stash_bytes < encoder_stash_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "encoder stash too small");
  StackStash cs;
  void* gemm; size_t gemm_bytes;
  Carve wc(ws);
  stack_ws_layout(wc, B, T, 3, kEncCh, false, &cs, &gemm, &gemm_bytes);
  float* rows;     // the last layer's output as plain rows
  if (a->stash) {
    const EncStash st = enc_stash(a->stash, B, T);
    cs = st.cs;
    T2_CUDA(cudaMemsetAsync(cs.x[0], 0, (char*)st.xl - (char*)cs.x[0], s));   // the conv stack, pad rows included
    rows = st.xl; *gates = st.gates; *cst = st.cst;
  } else {
    T2_CUDA(cudaMemsetAsync(cs.x[0], 0, (char*)cs.z[0] - (char*)cs.x[0], s));   // the activations, pad rows included
    rows = cs.x[3]; *gates = nullptr; *cst = nullptr;   // nothing reads x[3] as padded rows: it holds the plain ones
  }
  const long n = (long)B * T * kEnc;
  if (a->embedded)
    rows_to_padded_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->embedded, (long)T * kEnc, nullptr, cs.x[0], B, T, kEnc);
  else embed_to_padded_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->text, m->w[W_EMB], cs.x[0], B, T, m->cfg.n_symbols);
  T2_LAUNCH_CHECK();
  ConvLayer L[3];
  enc_layers(m, a->training, a->keep, B, T, L);
  for (int i = 0; i < 3; ++i) {
    float* yp = (i == 2 && !a->stash) ? nullptr : cs.x[i + 1];
    T2_TRY(conv_fwd(m, L[i], B, T, a->training, a->seed, cs.x[i], cs.z[i], cs.stats[i], yp, i == 2 ? rows : nullptr,
                    a->training != 0, cs.stats[i] + 2 * L[i].cout, gemm, gemm_bytes, s));
  }
  *xl = rows;
  return T2_OK;
}
// after the LSTM ran: keep a copy of the output for the backward pass
int encoder_stash_output(const T2EncoderArgs* a, cudaStream_t s) {
  const EncStash st = enc_stash(a->stash, a->B, a->T);
  T2_CUDA(cudaMemcpyAsync(st.mem, a->memory, (size_t)a->B * a->T * kEnc * 4, cudaMemcpyDeviceToDevice, s));
  return T2_OK;
}

constexpr int kEncBwdSplit = 8;   // K splits of the W_hh products in the reverse recurrence
struct EncBwdWs {
  float* dG;               // (B, T, 2 dirs, 1024)
  float *hp, *dxl;         // (B T, 512)
  float* part;             // (2, kEncBwdSplit, 64, 256)
  float* g_c;              // (2, 64, 256)
  float *gz, *gxa, *gxb;   // padded rows (B (T+4), 512)
  float *sums, *tmp;
  void* gemm; size_t gemm_bytes;   // scratch of the BiLSTM's weight / input gradient GEMMs and bias column sums
  ConvBwdWs cw;
};
static void encoder_backward_ws_layout(Carve& c, int B, int T, EncBwdWs* w) {
  const size_t Mp = (size_t)B * (T + 2 * kPadRows);
  w->dG = c.take<float>((size_t)B * T * 8 * kEncH);
  w->hp = c.take<float>((size_t)B * T * kEnc); w->dxl = c.take<float>((size_t)B * T * kEnc);
  w->part = c.take<float>((size_t)2 * kEncBwdSplit * 64 * kEncH);
  w->g_c = c.take<float>((size_t)2 * 64 * kEncH);
  w->gz = c.take<float>(Mp * kEnc); w->gxa = c.take<float>(Mp * kEnc); w->gxb = c.take<float>(Mp * kEnc);
  w->sums = c.take<float>((size_t)(2 + 2 * kRedSplit) * kEnc);
  w->tmp = c.take<float>(8 * kEncH);
  const int BT = B * T;
  w->gemm_bytes = std::max({gemm_tc_ws_bytes(4 * kEncH, kEnc, BT), gemm_tc_ws_bytes(4 * kEncH, kEncH, BT),
                            gemm_tc_ws_bytes(BT, kEnc, 4 * kEncH), colsum_ws_bytes(BT, 4 * kEncH)});
  w->gemm = c.take<char>(w->gemm_bytes);
  conv_bwd_layout(c, B, T, &w->cw);
}
size_t encoder_backward_ws_bytes(int B, int T) {
  Carve c(nullptr, 1024);
  EncBwdWs w;
  encoder_backward_ws_layout(c, B, T, &w);
  return c.bytes();
}

int encoder_backward(T2Model* m, const T2EncoderBwdArgs* a, cudaStream_t s) {
  const int B = a->B, T = a->T;
  constexpr int nsplit = kEncBwdSplit;
  if (B < 1 || B > 64) return fail(T2_ERR_UNSUPPORTED, "encoder backward: 1 <= B <= 64 (got %d)", B);
  if (a->n_grads != W_COUNT) return fail(T2_ERR_INVALID, "encoder backward: expected %d gradient pointers", (int)W_COUNT);
  if (a->ws_bytes < encoder_backward_ws_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "encoder backward workspace too small");
  if (a->stash_bytes < encoder_stash_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "encoder stash too small");
  const EncStash st = enc_stash(a->stash, B, T);
  EncBwdWs w;
  Carve wc(a->ws, 1024);
  encoder_backward_ws_layout(wc, B, T, &w);
  T2_CUDA(cudaMemsetAsync(w.g_c, 0, (size_t)2 * 64 * kEncH * 4, s));
  // ---- BiLSTM: reverse recurrence of both directions (model.py:169-171, 180-188) ----
  for (int step = 0; step < T; ++step) {
    enc_lstm_bwd_kernel<<<dim3(2, B), 256, 0, s>>>(a->d_memory, w.part, step > 0, st.gates, st.cst, a->lengths, w.g_c, w.dG, B, T, step, nsplit);
    T2_LAUNCH_CHECK();
    if (step + 1 < T) {
      enc_whh_bwd_kernel<<<dim3(2, nsplit, 2), 256, 0, s>>>(w.dG, m->w[W_ENC_LSTM + 1], m->w[W_ENC_LSTM + 5], w.part, B, T, step, nsplit);
      T2_LAUNCH_CHECK();
    }
  }
  float* const* G = a->grads;
  const int BT = B * T;
  const long n = (long)BT * kEnc;
  enc_hprev_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st.mem, w.hp, B, T);
  T2_LAUNCH_CHECK();
  for (int dir = 0; dir < 2; ++dir) {
    const int wb = W_ENC_LSTM + 4 * dir;
    const float* dGd = w.dG + (size_t)dir * 4 * kEncH;          // rows (b, t), row stride 2048
    if (G[wb])
      T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, true, false, 4 * kEncH, kEnc, BT, dGd, 8 * kEncH, st.xl, kEnc, G[wb],
                        kEnc, 0.f));
    if (G[wb + 1])
      T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, true, false, 4 * kEncH, kEncH, BT, dGd, 8 * kEncH,
                        w.hp + (size_t)dir * kEncH, kEnc, G[wb + 1], kEncH, 0.f));
    if (G[wb + 2] || G[wb + 3]) {
      T2_TRY(colsum_f32(s, w.gemm, w.gemm_bytes, dGd, 8 * kEncH, BT, 4 * kEncH, w.tmp));
      if (G[wb + 2]) T2_CUDA(cudaMemcpyAsync(G[wb + 2], w.tmp, 4 * kEncH * 4, cudaMemcpyDeviceToDevice, s));
      if (G[wb + 3]) T2_CUDA(cudaMemcpyAsync(G[wb + 3], w.tmp, 4 * kEncH * 4, cudaMemcpyDeviceToDevice, s));
    }
    // gradient wrt the LSTM input: dG_dir (BT x 1024) . W_ih_dir (1024 x 512)
    T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, false, false, BT, kEnc, 4 * kEncH, dGd, 8 * kEncH, m->w[wb], kEnc, w.dxl,
                      kEnc, dir ? 1.f : 0.f));
  }
  // ---- conv stack ----
  ConvLayer L[3];
  enc_layers(m, a->training, a->keep, B, T, L);
  const float* g = w.dxl; int g_padded = 0;
  float* gx = w.gxa;
  for (int i = 2; i >= 0; --i) {
    const bool need_gx = i > 0 || a->d_embedded || (a->text && G[W_EMB]);
    T2_TRY(conv_bwd(m, L[i], B, T, a->training, a->seed, g, g_padded, st.cs.x[i], st.cs.z[i], st.cs.stats[i], st.cs.x[i + 1], w.gz,
                    need_gx ? gx : nullptr, w.sums, G, w.cw, s));
    g = gx; g_padded = 1;
    gx = gx == w.gxa ? w.gxb : w.gxa;
  }
  if (a->d_embedded) {
    padded_to_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(g, nullptr, a->d_embedded, B, T, kEnc);
    T2_LAUNCH_CHECK();
  }
  if (a->text && G[W_EMB]) {
    if ((size_t)B * T * sizeof(int) > 200 * 1024) return fail(T2_ERR_UNSUPPORTED, "encoder backward: B * T too large for the embedding kernel");
    T2_CUDA(cudaFuncSetAttribute(embed_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)B * T * sizeof(int))));
    embed_bwd_kernel<<<m->cfg.n_symbols, 256, (size_t)B * T * sizeof(int), s>>>(a->text, g, G[W_EMB], B, T, m->cfg.n_symbols);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

}  // namespace t2
