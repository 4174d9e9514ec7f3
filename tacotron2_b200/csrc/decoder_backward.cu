// Backward pass of the teacher-forced decoder (the autograd graph of Decoder.forward, model.py:381-416),
// fp32, derived by hand (tools/bwd_algorithm_check.py is the CPU statement of exactly this decomposition,
// checked against torch autograd through the oracle).
//
// Phase 1 (reverse time, 5 kernels per step; carries = gradients wrt the step-t states coming from t+1):
//   KA lstm_bwd_row : g_dh = carry + W_P^T [d_mel_t ; d_gate_t]  -> dropout mask -> LSTMCell backward -> dG_dec[t], g_dc
//   KB bwd_gemm_run : [g_ah | g_ctx | g_dh'] partials = dG_dec[t] . [W_ih^d | W_hh^d]      (model.py:366-369)
//   KC attention    : g_ctx total -> g_aw -> softmax backward -> g_s = g_e v (1 - tanh^2) -> g_q, g_pm (stashed),
//                     location layer backward -> carries for aw_{t-1}, awc_{t-1}          (model.py:43-86)
//   KD lstm_bwd_row : g_ah = carry + dG_dec part + g_q W_q -> mask -> LSTMCell backward    -> dG_att[t], g_ac
//   KE bwd_gemm_run : [g_x2 | g_ctx' | g_ah'] partials = dG_att[t] . [W_ih^a | W_hh^a]    (model.py:352-354)
// KB / KE are the wgmma split-fp16 skinny GEMM: kBwdGemmSplit partial sums over the reduction, summed by the consumer.
// Phase 2 (time batched, on the tensor-core GEMMs wgrad_tc / gemm_tc): every weight gradient is dG^T . X over all
// T x B rows; d_memory = d_pm W_m + sum_t aw_t (x) g_ctx_t.
#include <string.h>

#include <algorithm>

#include "decoder.h"
#include "gemm_f32.cuh"
#include "umma.cuh"
#include "gemm_tc.h"
#include "wgrad_tc.h"

namespace t2 {

namespace {

constexpr int kPBld = 1536 + 1024;   // [g_ah (1024) | g_ctx (512) | g_dh' (1024)]
constexpr int kPEld = 768 + 1024;    // [g_x2 (256) | g_ctx' (512) | g_ah' (1024)]
constexpr int kTaps = 2 * kLocK;     // 62 taps of the fused location filter
constexpr int kColsLd = 64;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// LSTMCell backward for one step (KA / KD).  grid B, block 1024: block = one batch row, thread = one hidden unit.
// ---------------------------------------------------------------------------------------------
struct LstmBwdArgs {
  // g_h = sum over sources of sum_s src[(s * 64 + b) * ld + off + unit]  +  sum_o vec[b][o] * Wv[o][unit]
  const float* src0; int ld0, off0, ns0;
  const float* src1; int ld1, off1, ns1;
  const float* add; int ldadd;             // (B, >= 1024) direct term or null
  const float* vec; int nvec, ldvec;       // (B, nvec) rows, row stride ldvec
  const float* Wv; int ldwv;               // (nvec, >= 1024)
  const uint8_t* keep;                     // (B, 1024) of this step or null
  int dropout; uint64_t seed; uint32_t site; float p;
  const float* gates;                      // (B, 4096) activations of this step
  const float* c; const float* c_prev;     // (B, 1024)
  float* g_c;                              // (B, 1024) carry, in/out
  float* dG;                               // (B, 4096) out
  uint8_t* img; float* inv_scale;          // scaled split-fp16 operand image of dG + 1/scale per row
};

// The block knows the row maximum of dG, scales the row by a power of two into [0.5, 1) and writes it as the
// split-fp16 operand image of the tensor-core GEMM (gradients span many orders of magnitude; fp16 does not) next to
// the fp32 copy.
__global__ void __launch_bounds__(1024) lstm_bwd_row_kernel(const LstmBwdArgs a) {
  __shared__ float s_vec[128];
  __shared__ float s_max[32];
  const int b = blockIdx.x, unit = threadIdx.x;
  for (int i = threadIdx.x; i < a.nvec; i += 1024) s_vec[i] = a.vec[(long)b * a.ldvec + i];
  __syncthreads();
  float g_h = a.add ? a.add[(long)b * a.ldadd + unit] : 0.f;
  if (a.src0) {
#pragma unroll 4
    for (int s = 0; s < a.ns0; ++s) g_h += a.src0[((long)s * 64 + b) * a.ld0 + a.off0 + unit];
  }
  if (a.src1) {
#pragma unroll 4
    for (int s = 0; s < a.ns1; ++s) g_h += a.src1[((long)s * 64 + b) * a.ld1 + a.off1 + unit];
  }
  {
    float p4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
    for (int o = 0; o < a.nvec; o += 4) {
#pragma unroll
      for (int i = 0; i < 4; ++i) p4[i] = fmaf(s_vec[o + i], __ldg(a.Wv + (long)(o + i) * a.ldwv + unit), p4[i]);
    }
    g_h += (p4[0] + p4[1]) + (p4[2] + p4[3]);
  }
  if (a.dropout) {
    const long idx = (long)b * 1024 + unit;
    const bool keep = a.keep ? a.keep[idx] != 0 : philox_keep(a.seed, a.site, (uint64_t)idx, a.p);
    g_h = keep ? g_h * (1.f / (1.f - a.p)) : 0.f;
  }
  const float* gp = a.gates + (long)b * 4096 + unit;
  const float gi = gp[0], gf = gp[1024], gg = gp[2048], go = gp[3072];
  const float c = a.c[(long)b * 1024 + unit], cp = a.c_prev[(long)b * 1024 + unit];
  const float tc = tanhf(c);
  const float d_o = g_h * tc;
  const float d_c = a.g_c[(long)b * 1024 + unit] + g_h * go * (1.f - tc * tc);
  float d[4];
  d[0] = d_c * gg * gi * (1.f - gi);
  d[1] = d_c * cp * gf * (1.f - gf);
  d[2] = d_c * gi * (1.f - gg * gg);
  d[3] = d_o * go * (1.f - go);
  float* dg = a.dG + (long)b * 4096 + unit;
#pragma unroll
  for (int g = 0; g < 4; ++g) dg[g * 1024] = d[g];
  a.g_c[(long)b * 1024 + unit] = d_c * gf;
  // row maximum -> power-of-two scale
  float mx = fmaxf(fmaxf(fabsf(d[0]), fabsf(d[1])), fmaxf(fabsf(d[2]), fabsf(d[3])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = s_max[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  int e = 0;
  if (mx > 0.f && mx < 3.0e38f) frexpf(mx, &e);           // mx = f * 2^e, f in [0.5, 1)
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  const float sc = ldexpf(1.f, -e);
  if (threadIdx.x == 0) a.inv_scale[b] = ldexpf(1.f, e);
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int k = g * 1024 + unit;
    __half h, l;
    split_fp16(d[g] * sc, h, l);
    __half* hi = reinterpret_cast<__half*>(a.img + (size_t)(k >> 6) * 16384);
    __half* lo = hi + 64 * kChunkK;
    const uint32_t eo = img_elem_offset(b, k & 63);
    hi[eo] = h; lo[eo] = l;
  }
}

// ---------------------------------------------------------------------------------------------
// Attention backward for one step (KC).  grid (2, B): CTA (h, b) handles attention dims [64h, 64h + 64) of row b.
// ---------------------------------------------------------------------------------------------
struct AttBwdArgs {
  int t, T, B, Te, carry;                 // carry = (t < T - 1)
  const int32_t* len;
  const float* memory; const float* pm; const float* q;   // (B,Te,512), (B,Te,128), (T,B,128)
  const float* v; const float* weff;      // (128), (128, 62)
  const float* align; const float* awc;   // (B,T,Te) forward weights / cumulative weights BEFORE step t
  const float* d_align;                   // (B,T,Te) or null
  const float* PE; const float* PB;       // partials of step t+1 (KE) and of this step (KB)
  int nsE, nsB;                           // number of partial sums in PE / PB
  const float* gproj;                     // (T,B,1536) = [d_mel_t ; d_gate_t] . W_PG, all steps (time batched)
  const float* weffT;                     // (62, 128) transposed fused location filter
  float* dctx; float* dx2; float* dq;     // (T,B,512), (T,B,256), (T,B,128)
  float* gs;                              // (T,B,Te,128)
  float* gcat;                            // (2 pingpong, 2 halves, B, 2, Te)
  float* cacc;                            // (2 pingpong, B, Te)
  float* dv;                              // (B, 128) accumulated
};

constexpr int kAttT = 512;               // threads of att_bwd_kernel: 16 warps hide the global-load latency
constexpr int kAttG = kAttT / 64;         // position groups in steps (4), (5)
__global__ void __launch_bounds__(kAttT) att_bwd_kernel(const AttBwdArgs a) {
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.x, b = blockIdx.y;
  const int t = a.t, T = a.T, B = a.B, Te = a.Te;
  const int TeP = Te + kLocK - 1;
  float* s_ctx = sm;                       // 512
  float* s_dy = s_ctx + 512;               // 96
  float* s_red = s_dy + 96;                // 64 + kAttG * 64 * 2
  float* s_aw = s_red + 64 + kAttG * 128;          // Te (padded to 4)
  const int Te4 = (Te + 3) & ~3;
  float* s_ge = s_aw + Te4;                // Te
  float* s_pad0 = s_ge + Te4;              // TeP (+ slack)
  const int TeP4 = (TeP + 7) & ~3;
  float* s_pad1 = s_pad0 + TeP4;
  float* s_gs = s_pad1 + TeP4;             // Te4 x 64
  float* s_u = s_gs + (size_t)Te4 * 64;    // Te x 65
  const int rd = (t + 1) & 1, wr = t & 1;

  // previous / cumulative attention weights of this step (zero padded by 15 each side)   model.py:358-360
  for (int i = tid; i < TeP4; i += kAttT) { s_pad0[i] = 0.f; s_pad1[i] = 0.f; }
  __syncthreads();
  for (int j = tid; j < Te; j += kAttT) {
    s_pad0[15 + j] = t > 0 ? a.align[((long)b * T + t - 1) * Te + j] : 0.f;
    s_pad1[15 + j] = a.awc[((long)b * T + t) * Te + j];
    s_aw[j] = a.align[((long)b * T + t) * Te + j];
    // carries into aw_t: location conv of step t+1 (channel 0) and the cumulative weights (channel 1 + running sum)
    float g = 0.f, cv = 0.f;
    if (a.carry) {
      const float* g0 = a.gcat + (((long)rd * 2 + 0) * B + b) * 2 * Te;
      const float* g1 = a.gcat + (((long)rd * 2 + 1) * B + b) * 2 * Te;
      g = g0[j] + g1[j];
      cv = a.cacc[((long)rd * B + b) * Te + j] + g0[Te + j] + g1[Te + j];
    }
    if (h == 0) a.cacc[((long)wr * B + b) * Te + j] = cv;
    g += cv;
    if (a.d_align) g += a.d_align[((long)b * T + t) * Te + j];
    s_ge[j] = g;
  }
  // (1) total gradient wrt ctx_t: carry from step t+1's attention LSTM input, decoder LSTM input, projection
  for (int c = tid; c < 512; c += kAttT) {
    float g = a.gproj[((long)t * B + b) * 1536 + 1024 + c];
    if (a.carry) {
#pragma unroll 5
      for (int s = 0; s < a.nsE; ++s) g += a.PE[((long)s * 64 + b) * kPEld + 256 + c];
    }
#pragma unroll 4
    for (int s = 0; s < a.nsB; ++s) g += a.PB[((long)s * 64 + b) * kPBld + 1024 + c];
    s_ctx[c] = g;
    if (h == 0) a.dctx[((long)t * B + b) * 512 + c] = g;
  }
  if (h == 0 && a.carry && tid < 256) {   // gradient wrt the prenet output of step t+1 (first 256 columns of KE's result)
    float g = 0.f;
#pragma unroll 5
    for (int s = 0; s < a.nsE; ++s) g += a.PE[((long)s * 64 + b) * kPEld + tid];
    a.dx2[((long)(t + 1) * B + b) * 256 + tid] = g;
  }
  __syncthreads();
  // (2) g_aw[j] += memory[j] . g_ctx   (4 rows per warp iteration: 16 independent 16-byte loads in flight)  model.py:83-84
  {
    float4 gc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) gc[i] = *reinterpret_cast<const float4*>(s_ctx + (i * 32 + lane) * 4);
    for (int j0 = warp * 8; j0 < Te; j0 += 8 * (kAttT / 32)) {
      float acc[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        acc[r] = 0.f;
        const int j = j0 + r < Te ? j0 + r : Te - 1;
        const float4* mr = reinterpret_cast<const float4*>(a.memory + ((long)b * Te + j) * 512);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 m = __ldg(mr + i * 32 + lane);
          acc[r] += m.x * gc[i].x + m.y * gc[i].y + m.z * gc[i].z + m.w * gc[i].w;
        }
      }
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float v = warp_sum(acc[r]);
        if (lane == 0 && j0 + r < Te) s_ge[j0 + r] += v;
      }
    }
  }
  __syncthreads();
  // (3) softmax backward: g_e = aw * (g_aw - sum_j aw g_aw)                              model.py:82
  {
    float p = 0.f;
    for (int j = tid; j < Te; j += kAttT) p += s_aw[j] * s_ge[j];
    p = warp_sum(p);
    if (lane == 0) s_red[warp] = p;
    __syncthreads();
    float dot = 0.f;
#pragma unroll
    for (int w = 0; w < kAttT / 32; ++w) dot += s_red[w];
    __syncthreads();
    for (int j = tid; j < Te; j += kAttT) s_ge[j] = s_aw[j] * (s_ge[j] - dot);
    __syncthreads();
  }
  // (4) recompute s = q + pa + pm, g_s = g_e v (1 - tanh^2 s); thread = (attention dim, group of positions)
  {
    const int al = tid & 63, jg = tid >> 6, ag = h * 64 + al;
    float w[kTaps];
#pragma unroll
    for (int k = 0; k < kTaps; ++k) w[k] = __ldg(a.weffT + (long)k * kAtt + ag);
    const float qv = a.q[((long)t * B + b) * 128 + ag];
    const float vv = __ldg(a.v + ag);
    float gq = 0.f, dv = 0.f;
    for (int j0 = jg * 4; j0 < Te; j0 += 4 * kAttG) {
      float pa[4] = {0.f, 0.f, 0.f, 0.f}, pmv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pmv[i] = j0 + i < Te ? __ldg(a.pm + ((long)b * Te + j0 + i) * 128 + ag) : 0.f;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float* pad = (c == 0 ? s_pad0 : s_pad1) + j0;
        float w0 = pad[0], w1 = pad[1], w2 = pad[2], w3 = pad[3];
#pragma unroll
        for (int k = 0; k < kLocK; ++k) {
          const float wk = w[c * kLocK + k];
          pa[0] = fmaf(wk, w0, pa[0]); pa[1] = fmaf(wk, w1, pa[1]); pa[2] = fmaf(wk, w2, pa[2]); pa[3] = fmaf(wk, w3, pa[3]);
          w0 = w1; w1 = w2; w2 = w3; w3 = pad[k + 4];
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = j0 + i;
        if (j < Te) {
          const float s = qv + pa[i] + pmv[i];
          const float th = tanhf(s);
          const float ge = s_ge[j];
          const float g = ge * vv * (1.f - th * th);
          dv = fmaf(ge, th, dv);
          gq += g;
          s_gs[j * 64 + al] = g;
          a.gs[(((long)t * B + b) * Te + j) * 128 + ag] = g;
        }
      }
    }
    s_red[64 + (jg * 64 + al) * 2 + 0] = gq;
    s_red[64 + (jg * 64 + al) * 2 + 1] = dv;
    __syncthreads();
    if (tid < 64) {
      float gq4 = 0.f, dv4 = 0.f;
#pragma unroll
      for (int g = 0; g < kAttG; ++g) { gq4 += s_red[64 + (g * 64 + tid) * 2]; dv4 += s_red[64 + (g * 64 + tid) * 2 + 1]; }
      a.dq[((long)t * B + b) * 128 + h * 64 + tid] = gq4;
      a.dv[(long)b * 128 + h * 64 + tid] += dv4;
    }
  }
  // (5) U[j][ck] = sum_a g_s[j][a] Weff[a][ck]  (this half's 64 attention dims)
  {
    const int ck = tid & 63, jg = tid >> 6;
    float wc[64];
#pragma unroll
    for (int al = 0; al < 64; ++al) wc[al] = ck < kTaps ? __ldg(a.weff + (long)(h * 64 + al) * kTaps + ck) : 0.f;
    for (int j = jg; j < Te; j += kAttG) {
      const float4* g4 = reinterpret_cast<const float4*>(s_gs + j * 64);
      float u = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 g = g4[i];
        u = fmaf(g.x, wc[i * 4], u); u = fmaf(g.y, wc[i * 4 + 1], u); u = fmaf(g.z, wc[i * 4 + 2], u); u = fmaf(g.w, wc[i * 4 + 3], u);
      }
      s_u[j * 65 + ck] = u;
    }
  }
  __syncthreads();
  // (6) transposed location conv: g_cat[c][j'] = sum_k U[j' + 15 - k][c * 31 + k]        model.py:23
  for (int i = tid; i < 2 * Te; i += kAttT) {
    const int c = i / Te, jp = i - c * Te;
    float g = 0.f;
    for (int k = 0; k < kLocK; ++k) {
      const int j = jp + 15 - k;
      if (j >= 0 && j < Te) g += s_u[j * 65 + c * kLocK + k];
    }
    a.gcat[(((long)wr * 2 + h) * B + b) * 2 * Te + i] = g;
  }
}

size_t att_bwd_smem(int Te) {
  const int Te4 = (Te + 3) & ~3, TeP4 = (Te + kLocK - 1 + 7) & ~3;
  return (size_t)(512 + 96 + 64 + kAttG * 128 + 2 * Te4 + 2 * TeP4 + (size_t)Te4 * 64 + (size_t)Te * 65 + 16) * sizeof(float);
}

// ---- small helper kernels -------------------------------------------------------------------
__global__ void dy_kernel(const float* __restrict__ d_mel, const float* __restrict__ d_gate, float* __restrict__ dY, int B, int T) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)T * B * 81) return;
  const int o = (int)(i % 81); const long r = i / 81; const int b = (int)(r % B); const int t = (int)(r / B);
  dY[i] = o < 80 ? d_mel[((long)b * T + t) * 80 + o] : d_gate[(long)b * T + t];
}
__global__ void awc_kernel(const float* __restrict__ align, float* __restrict__ awc, int B, int T, int Te) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Te) return;
  const int b = i / Te, j = i - b * Te;
  float run = 0.f;
  for (int t = 0; t < T; ++t) {
    awc[((long)b * T + t) * Te + j] = run;                 // cumulative weights BEFORE step t (model.py:365)
    run += align[((long)b * T + t) * Te + j];
  }
}
__global__ void weff_kernel(const float* __restrict__ wld, const float* __restrict__ wloc, float* __restrict__ weff,
                            float* __restrict__ weffT) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // Weff[a][c*31+k] = sum_f W_ld[a][f] W_loc[f][c][k]
  if (i >= kAtt * kTaps) return;
  const int a = i / kTaps, ck = i - a * kTaps;
  float s = 0.f;
  for (int f = 0; f < kLocF; ++f) s = fmaf(wld[a * kLocF + f], wloc[f * kTaps + ck], s);
  weff[i] = s;
  weffT[(long)ck * kAtt + a] = s;
}
__global__ void dweff_split_kernel(const float* __restrict__ dweff, const float* __restrict__ wld, const float* __restrict__ wloc,
                                   float* __restrict__ d_wld, float* __restrict__ d_wloc) {
  // dWeff (128, ld 64) -> dW_ld[a][f] = sum_ck dWeff[a][ck] W_loc[f][ck] ;  dW_loc[f][ck] = sum_a W_ld[a][f] dWeff[a][ck]
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kAtt * kLocF && d_wld) {
    const int a = i / kLocF, f = i - a * kLocF;
    float s = 0.f;
    for (int ck = 0; ck < kTaps; ++ck) s = fmaf(dweff[a * kColsLd + ck], wloc[f * kTaps + ck], s);
    d_wld[i] = s;
  }
  if (i < kLocF * kTaps && d_wloc) {
    const int f = i / kTaps, ck = i - f * kTaps;
    float s = 0.f;
    for (int a = 0; a < kAtt; ++a) s = fmaf(wld[a * kLocF + f], dweff[a * kColsLd + ck], s);
    d_wloc[i] = s;
  }
}
__global__ void im2col_kernel(const float* __restrict__ align, const float* __restrict__ awc, float* __restrict__ cols,
                              int B, int T, int Te) {
  // cols[(t, b, j)][c * 31 + k] = (c == 0 ? aw_{t-1} : awc_{t-1})[j + k - 15], zero outside; columns 62, 63 = 0
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)T * B * Te * kColsLd) return;
  const int ck = (int)(i & 63); const long r = i >> 6;
  const int j = (int)(r % Te); const long tb = r / Te; const int b = (int)(tb % B); const int t = (int)(tb / B);
  float v = 0.f;
  if (ck < kTaps) {
    const int c = ck / kLocK, k = ck - c * kLocK, jj = j + k - 15;
    if (jj >= 0 && jj < Te) v = c == 0 ? (t > 0 ? align[((long)b * T + t - 1) * Te + jj] : 0.f) : awc[((long)b * T + t) * Te + jj];
  }
  cols[i] = v;
}
__global__ void reduce_pe_x2_kernel(const float* __restrict__ PE, float* __restrict__ dx2, int B, int nsE) {
  const int b = blockIdx.x, c = threadIdx.x;   // step 0: g_x2 = sum of the partials
  if (b >= B) return;
  float g = 0.f;
  for (int s = 0; s < nsE; ++s) g += PE[((long)s * 64 + b) * kPEld + c];
  dx2[(long)b * 256 + c] = g;
}
__global__ void fill_kernel(float* p, float v, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void sum_rows_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // out[i] = sum_r x[r][i]  (small row counts)
  if (i >= n) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[(long)r * n + i];
  out[i] = s;
}
__global__ void prenet_dz_kernel(const float* g, const float* __restrict__ act, float* out, long n) {
  // dropout(p = 0.5) o relu backward: dz = 2 g where the (already masked) activation is positive   model.py:99
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = act[i] > 0.f ? 2.f * g[i] : 0.f;
}

struct BwdWs {
  float *dga, *dgd, *q, *dq, *awc, *pm, *dpm, *dctx, *dy, *gs, *cols, *pb, *pe, *gdc, *gac, *cacc, *gcat, *dv, *weff, *dweff,
      *tmp, *gproj, *weffT, *inv_scale;
  uint8_t *img_d, *img_a; DecoderCtrl* ctrl;
  uint8_t* bwd_wimg[2];                // W^T images of the skinny GEMMs (bwd_gemm_prepare)
  void* gemm; size_t gemm_bytes;       // scratch of the gemm_tc products and column sums, shared in stream order
  WgradWs wg;
};
void bwd_ws_layout(Carve& c, int B, int Te, int T, BwdWs* w) {
  const size_t TB = (size_t)T * B;
  w->dga = c.take<float>(TB * 4096); w->dgd = c.take<float>(TB * 4096);
  w->q = c.take<float>(TB * 128); w->dq = c.take<float>(TB * 128);
  w->awc = c.take<float>((size_t)B * T * Te);
  w->pm = c.take<float>((size_t)B * Te * 128); w->dpm = c.take<float>((size_t)B * Te * 128);
  w->dctx = c.take<float>(TB * 512); w->dy = c.take<float>(TB * 81);
  w->gs = c.take<float>(TB * Te * 128); w->cols = c.take<float>(TB * Te * kColsLd);
  w->pb = c.take<float>((size_t)kBwdGemmSplit * 64 * kPBld); w->pe = c.take<float>((size_t)kBwdGemmSplit * 64 * kPEld);
  w->gdc = c.take<float>((size_t)64 * 1024); w->gac = c.take<float>((size_t)64 * 1024);
  w->cacc = c.take<float>((size_t)2 * B * Te); w->gcat = c.take<float>((size_t)2 * 2 * B * 2 * Te);
  w->dv = c.take<float>((size_t)B * 128);
  w->weff = c.take<float>((size_t)kAtt * kTaps); w->dweff = c.take<float>((size_t)kAtt * kColsLd);
  w->tmp = c.take<float>(4096);
  w->gproj = c.take<float>(TB * 1536); w->weffT = c.take<float>((size_t)kAtt * kTaps);
  w->inv_scale = c.take<float>(128);
  w->img_d = c.take<uint8_t>(kBwdImgBytes, 1024); w->img_a = c.take<uint8_t>(kBwdImgBytes, 1024);
  w->ctrl = c.take<DecoderCtrl>(1);
  for (int i = 0; i < 2; ++i) w->bwd_wimg[i] = c.take<uint8_t>(bwd_wimg_bytes(i), 1024);
  const int BTe = B * Te, TBi = (int)TB;
  w->gemm_bytes = std::max({gemm_tc_ws_bytes(BTe, kAtt, kEnc), gemm_tc_ws_bytes(TBi, kAtt, kARnn),
                            gemm_tc_ws_bytes(TBi, kDRnn + kEnc, 81), gemm_tc_ws_bytes(kMel, kDRnn, TBi),
                            gemm_tc_ws_bytes(kMel, kEnc, TBi), gemm_tc_ws_bytes(1, kDRnn, TBi), gemm_tc_ws_bytes(1, kEnc, TBi),
                            colsum_ws_bytes(TBi, 81), gemm_tc_ws_bytes(kAtt, kARnn, TBi),
                            gemm_tc_ws_bytes(kAtt, kColsLd, (int)(TB * Te)), colsum_ws_bytes(T, BTe * kAtt),
                            gemm_tc_ws_bytes(kAtt, kEnc, BTe), gemm_tc_ws_bytes(BTe, kEnc, kAtt), gemm_tc_ws_bytes(Te, kEnc, T, B)});
  w->gemm = c.take<char>(w->gemm_bytes);
  wgrad_tc_layout(c, T, &w->wg);
}

}  // namespace

size_t decoder_backward_ws_bytes(int B, int T_enc, int T_mel) {
  Carve c(nullptr, 1024);
  BwdWs w;
  bwd_ws_layout(c, B, T_enc, T_mel, &w);
  return c.bytes();
}

int decoder_backward(T2Model* m, const T2DecoderBwdArgs* a, cudaStream_t s) {
  const int B = a->B, Te = a->T_enc, T = a->T_mel;
  if (B < 1 || B > 64) return fail(T2_ERR_UNSUPPORTED, "decoder backward: 1 <= B <= 64 (got %d)", B);
  if (Te < 1 || T < 1) return fail(T2_ERR_INVALID, "decoder backward: bad sizes");
  const size_t smem = att_bwd_smem(Te);
  if (smem > 220 * 1024) return fail(T2_ERR_UNSUPPORTED, "decoder backward: T_enc = %d too long for the attention kernel", Te);
  if (a->n_grads != W_COUNT) return fail(T2_ERR_INVALID, "decoder backward: expected %d gradient pointers", (int)W_COUNT);
  if (a->ws_bytes < decoder_backward_ws_bytes(B, Te, T)) return fail(T2_ERR_WORKSPACE, "decoder backward workspace too small");
  if (a->stash_bytes < decoder_stash_bytes(B, T)) return fail(T2_ERR_WORKSPACE, "decoder stash too small");
  DecoderStash st;
  Carve sc(const_cast<void*>(a->stash));
  decoder_stash_layout(sc, B, T, &st);
  BwdWs w;
  Carve wc(a->ws, 1024);
  bwd_ws_layout(wc, B, Te, T, &w);
  const size_t TB = (size_t)T * B;
  const int training = a->training;
  const float p_att = m->cfg.p_attention_dropout, p_dec = m->cfg.p_decoder_dropout;

  // ---- set-up -------------------------------------------------------------------------------------
  T2_CUDA(cudaMemsetAsync(w.gdc, 0, (size_t)64 * 1024 * 4, s));
  T2_CUDA(cudaMemsetAsync(w.gac, 0, (size_t)64 * 1024 * 4, s));
  T2_CUDA(cudaMemsetAsync(w.dv, 0, (size_t)B * 128 * 4, s));
  T2_CUDA(cudaMemsetAsync(w.cacc, 0, (size_t)2 * B * Te * 4, s));
  T2_CUDA(cudaMemsetAsync(w.gcat, 0, (size_t)8 * B * Te * 4, s));
  {
    const long n = (long)TB * 81;
    dy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->d_mel, a->d_gate, w.dy, B, T);
    T2_LAUNCH_CHECK();
    awc_kernel<<<(B * Te + 127) / 128, 128, 0, s>>>(a->align, w.awc, B, T, Te);
    T2_LAUNCH_CHECK();
    weff_kernel<<<(kAtt * kTaps + 255) / 256, 256, 0, s>>>(m->w[W_ATT_LOC_DENSE], m->w[W_ATT_LOC_CONV], w.weff, w.weffT);
    T2_LAUNCH_CHECK();
  }
  // processed_memory (model.py:288) and the processed queries of all steps (model.py:57)
  const int sms = m->sm_count;
  T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, false, true, B * Te, kAtt, kEnc, a->memory, kEnc, m->w[W_ATT_MEMORY], kEnc, w.pm,
                    kAtt, 0.f));
  T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, false, true, (int)TB, kAtt, kARnn, st.ha + (size_t)B * kARnn, kARnn,
                    m->w[W_ATT_QUERY], kARnn, w.q, kAtt, 0.f));
  // projection / gate contribution to g_dh and g_ctx of every step: [d_mel_t ; d_gate_t] . [W_proj ; W_gate]  (model.py:373-378)
  T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, false, false, (int)TB, kDRnn + kEnc, 81, w.dy, 81, m->projgate_w, kDRnn + kEnc,
                    w.gproj, kDRnn + kEnc, 0.f));
  T2_CUDA(cudaFuncSetAttribute(att_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // skinny GEMMs (KB / KE): weight images, zeroed operand images, control block and unit scales
  T2_TRY(bwd_gemm_prepare(m, w.bwd_wimg, s));
  T2_CUDA(cudaMemsetAsync(w.img_d, 0, kBwdImgBytes, s));      // rows >= B stay zero
  T2_CUDA(cudaMemsetAsync(w.img_a, 0, kBwdImgBytes, s));
  T2_CUDA(cudaMemsetAsync(w.ctrl, 0, sizeof(DecoderCtrl), s));
  fill_kernel<<<1, 128, 0, s>>>(w.inv_scale, 1.f, 128);
  T2_LAUNCH_CHECK();
  // ---- phase 1: reverse-time recurrence ---------------------------------------------------------------
  for (int t = T - 1; t >= 0; --t) {
    const int carry = t < T - 1;
    {  // KA
      LstmBwdArgs k;
      memset(&k, 0, sizeof(k));
      k.src0 = carry ? w.pb : nullptr; k.ld0 = kPBld; k.off0 = 1536; k.ns0 = kBwdGemmSplit;
      k.add = w.gproj + (size_t)t * B * 1536; k.ldadd = 1536;
      k.img = w.img_d; k.inv_scale = w.inv_scale;
      k.keep = a->dec_keep ? a->dec_keep + (size_t)t * B * kDRnn : nullptr;
      k.dropout = training; k.seed = a->seed; k.site = (uint32_t)(t * 4 + 3); k.p = p_dec;
      k.gates = st.gd + (size_t)t * B * 4096; k.c = st.cd + (size_t)(t + 1) * B * kDRnn; k.c_prev = st.cd + (size_t)t * B * kDRnn;
      k.g_c = w.gdc; k.dG = w.dgd + (size_t)t * B * 4096;
      lstm_bwd_row_kernel<<<B, 1024, 0, s>>>(k);
      T2_LAUNCH_CHECK();
    }
    T2_TRY(bwd_gemm_run(m, 0, w.bwd_wimg[0], w.img_d, w.inv_scale, w.pb, kPBld, w.ctrl, s));   // KB
    {  // KC
      AttBwdArgs k;
      memset(&k, 0, sizeof(k));
      k.t = t; k.T = T; k.B = B; k.Te = Te; k.carry = carry; k.len = a->memory_lengths;
      k.memory = a->memory; k.pm = w.pm; k.q = w.q; k.v = m->w[W_ATT_V]; k.weff = w.weff;
      k.align = a->align; k.awc = w.awc; k.d_align = a->d_align;
      k.PE = w.pe; k.PB = w.pb; k.nsE = kBwdGemmSplit; k.nsB = kBwdGemmSplit; k.gproj = w.gproj; k.weffT = w.weffT;
      k.dctx = w.dctx; k.dx2 = a->d_prenet; k.dq = w.dq; k.gs = w.gs; k.gcat = w.gcat; k.cacc = w.cacc; k.dv = w.dv;
      att_bwd_kernel<<<dim3(2, B), kAttT, smem, s>>>(k);
      T2_LAUNCH_CHECK();
    }
    {  // KD
      LstmBwdArgs k;
      memset(&k, 0, sizeof(k));
      k.src0 = carry ? w.pe : nullptr; k.ld0 = kPEld; k.off0 = 768; k.ns0 = kBwdGemmSplit;
      k.src1 = w.pb; k.ld1 = kPBld; k.off1 = 0; k.ns1 = kBwdGemmSplit;
      k.img = w.img_a; k.inv_scale = w.inv_scale + 64;
      k.vec = w.dq + (size_t)t * B * 128; k.nvec = 128; k.ldvec = 128; k.Wv = m->w[W_ATT_QUERY]; k.ldwv = kARnn;
      k.keep = a->att_keep ? a->att_keep + (size_t)t * B * kARnn : nullptr;
      k.dropout = training; k.seed = a->seed; k.site = (uint32_t)(t * 4 + 2); k.p = p_att;
      k.gates = st.ga + (size_t)t * B * 4096; k.c = st.ca + (size_t)(t + 1) * B * kARnn; k.c_prev = st.ca + (size_t)t * B * kARnn;
      k.g_c = w.gac; k.dG = w.dga + (size_t)t * B * 4096;
      lstm_bwd_row_kernel<<<B, 1024, 0, s>>>(k);
      T2_LAUNCH_CHECK();
    }
    T2_TRY(bwd_gemm_run(m, 1, w.bwd_wimg[1], w.img_a, w.inv_scale + 64, w.pe, kPEld, w.ctrl, s));   // KE
  }
  reduce_pe_x2_kernel<<<B, 256, 0, s>>>(w.pe, a->d_prenet, B, kBwdGemmSplit);
  T2_LAUNCH_CHECK();

  // ---- phase 2: time-batched gradients --------------------------------------------------------------------
  float* const* G = a->grads;
  const int TBi = (int)TB;
  // LSTM weight / bias gradients on the time-batched wgrad_tc engine
  T2_TRY(wgrad_tc_run(m, B, T, w.dga, w.dgd, a->teacher_prenet, st, G, w.wg, s));
  // projection + gate on [dh_t | ctx_t]                                                   model.py:373-378
  if (G[W_PROJ_W]) {
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, kMel, kDRnn, TBi, w.dy, 81, st.hd + (size_t)B * kDRnn, kDRnn,
                      G[W_PROJ_W], kDRnn + kEnc, 0.f));
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, kMel, kEnc, TBi, w.dy, 81, st.ctx + (size_t)B * kEnc, kEnc,
                      G[W_PROJ_W] + kDRnn, kDRnn + kEnc, 0.f));
  }
  if (G[W_GATE_W]) {
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, 1, kDRnn, TBi, w.dy + 80, 81, st.hd + (size_t)B * kDRnn, kDRnn,
                      G[W_GATE_W], kDRnn + kEnc, 0.f));
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, 1, kEnc, TBi, w.dy + 80, 81, st.ctx + (size_t)B * kEnc, kEnc,
                      G[W_GATE_W] + kDRnn, kDRnn + kEnc, 0.f));
  }
  if (G[W_PROJ_B] || G[W_GATE_B]) {
    T2_TRY(colsum_f32(s, w.gemm, w.gemm_bytes, w.dy, 81, TBi, 81, w.tmp));
    if (G[W_PROJ_B]) T2_CUDA(cudaMemcpyAsync(G[W_PROJ_B], w.tmp, 80 * 4, cudaMemcpyDeviceToDevice, s));
    if (G[W_GATE_B]) T2_CUDA(cudaMemcpyAsync(G[W_GATE_B], w.tmp + 80, 4, cudaMemcpyDeviceToDevice, s));
  }
  if (G[W_ATT_QUERY])
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, kAtt, kARnn, TBi, w.dq, kAtt, st.ha + (size_t)B * kARnn, kARnn,
                      G[W_ATT_QUERY], kARnn, 0.f));
  if (G[W_ATT_V]) {
    sum_rows_kernel<<<1, 128, 0, s>>>(w.dv, G[W_ATT_V], B, 128);
    T2_LAUNCH_CHECK();
  }
  if (G[W_ATT_LOC_CONV] || G[W_ATT_LOC_DENSE]) {   // through the fused filter Weff = W_ld . W_loc   model.py:23-25
    const long n = (long)TB * Te * kColsLd;
    im2col_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->align, w.awc, w.cols, B, T, Te);
    T2_LAUNCH_CHECK();
    // K = T*B*Te rows in one call: the GEMM drains its accumulator every 64 rows and splits K over the SMs
    const int R = (int)((long)TB * Te);
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, kAtt, kColsLd, R, w.gs, kAtt, w.cols, kColsLd, w.dweff, kColsLd, 0.f));
    dweff_split_kernel<<<(kAtt * kLocF + 255) / 256, 256, 0, s>>>(w.dweff, m->w[W_ATT_LOC_DENSE], m->w[W_ATT_LOC_CONV],
                                                                  G[W_ATT_LOC_DENSE], G[W_ATT_LOC_CONV]);
    T2_LAUNCH_CHECK();
  }
  // d_pm = sum_t g_s[t]  -> memory_layer gradient and its share of d_memory              model.py:288
  T2_TRY(colsum_f32(s, w.gemm, w.gemm_bytes, w.gs, (long)B * Te * kAtt, T, B * Te * kAtt, w.dpm));
  if (G[W_ATT_MEMORY])
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, true, false, kAtt, kEnc, B * Te, w.dpm, kAtt, a->memory, kEnc, G[W_ATT_MEMORY],
                      kEnc, 0.f));
  if (a->d_memory) {
    T2_TRY(gemm_tc_rm(sms, s, w.gemm, w.gemm_bytes, false, false, B * Te, kEnc, kAtt, w.dpm, kAtt, m->w[W_ATT_MEMORY], kEnc,
                      a->d_memory, kEnc, 0.f));
    // + sum_t aw_t[b] (x) g_ctx_t[b]: per row b, (Te x T) . (T x 512)                      model.py:83-84
    GemmTc g;        // d_memory[b] (Te x 512) += align[b]^T (T x Te stored) . dctx[:, b, :] (T x 512, rows B * 512 apart)
    g.ta = true; g.tb = false; g.M = Te; g.N = kEnc; g.K = T;
    g.A = a->align; g.lda = Te; g.strideA = (long)T * Te;
    g.B = w.dctx; g.ldb = (long)B * kEnc; g.strideB = kEnc;
    g.C = a->d_memory; g.ldc = kEnc; g.strideC = (long)Te * kEnc; g.beta = 1.f; g.batch = B;
    g.ws = w.gemm; g.ws_bytes = w.gemm_bytes;
    T2_TRY(gemm_tc(sms, s, g));
  }
  return T2_OK;
}

// ---------------------------------------------------------------------------------------------
// Prenet backward (model.py:97-100): recompute both layers with the same masks, then two plain GEMMs each.
// ---------------------------------------------------------------------------------------------
struct PrenetBwdWs {
  float *x1, *x2, *dz2, *dz1;       // (M, 256) each
  void* gemm; size_t gemm_bytes;    // scratch of the three products
};
static void prenet_backward_ws_layout(Carve& c, int M, PrenetBwdWs* w) {
  w->x1 = c.take<float>((size_t)M * kPre); w->x2 = c.take<float>((size_t)M * kPre);
  w->dz2 = c.take<float>((size_t)M * kPre); w->dz1 = c.take<float>((size_t)M * kPre);
  w->gemm_bytes = std::max({gemm_tc_ws_bytes(kPre, kPre, M), gemm_tc_ws_bytes(M, kPre, kPre), gemm_tc_ws_bytes(kPre, kMel, M)});
  w->gemm = c.take<char>(w->gemm_bytes);
}
size_t prenet_backward_ws_bytes(int M) { Carve c(nullptr); PrenetBwdWs w; prenet_backward_ws_layout(c, M, &w); return c.bytes(); }

int prenet_backward(T2Model* m, const T2PrenetBwdArgs* a, cudaStream_t s) {
  const int M = a->M;
  if (a->n_grads != W_COUNT) return fail(T2_ERR_INVALID, "prenet backward: expected %d gradient pointers", (int)W_COUNT);
  if (a->ws_bytes < prenet_backward_ws_bytes(M)) return fail(T2_ERR_WORKSPACE, "prenet backward workspace too small");
  Carve c(a->ws);
  PrenetBwdWs w;
  prenet_backward_ws_layout(c, M, &w);
  GemmArgs g;
  g.seg[0] = {a->frames, kMel, m->w[W_PRENET0], kMel, kMel};
  g.M = M; g.N = kPre; g.C = w.x1; g.ldc = kPre; g.act = ACT_RELU; g.p_drop = 0.5f;
  if (a->keep) { g.keep = a->keep; g.ldkeep = kPre; } else { g.philox = 1; g.seed = a->seed; g.site = 0xA0; }
  T2_TRY(gemm_f32(g, s));
  GemmArgs h;
  h.seg[0] = {w.x1, kPre, m->w[W_PRENET1], kPre, kPre};
  h.M = M; h.N = kPre; h.C = w.x2; h.ldc = kPre; h.act = ACT_RELU; h.p_drop = 0.5f;
  if (a->keep) { h.keep = a->keep + (size_t)M * kPre; h.ldkeep = kPre; } else { h.philox = 1; h.seed = a->seed; h.site = 0xA1; }
  T2_TRY(gemm_f32(h, s));
  const long n = (long)M * kPre;
  prenet_dz_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a->d_out, w.x2, w.dz2, n);
  T2_LAUNCH_CHECK();
  if (a->grads[W_PRENET1])
    T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, true, false, kPre, kPre, M, w.dz2, kPre, w.x1, kPre, a->grads[W_PRENET1],
                      kPre, 0.f));
  // d_x1 = w.dz2 . W2  -> through dropout o relu of layer 1
  T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, false, false, M, kPre, kPre, w.dz2, kPre, m->w[W_PRENET1], kPre, w.dz1,
                    kPre, 0.f));
  prenet_dz_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.dz1, w.x1, w.dz1, n);
  T2_LAUNCH_CHECK();
  if (a->grads[W_PRENET0])
    T2_TRY(gemm_tc_rm(m->sm_count, s, w.gemm, w.gemm_bytes, true, false, kPre, kMel, M, w.dz1, kPre, a->frames, kMel,
                      a->grads[W_PRENET0], kMel, 0.f));
  return T2_OK;
}

}  // namespace t2
