// WaveGlow inference (waveglow/glow.py:251-293, WaveGlow.infer) on sm_90a.
//
// Every dense product is one implicit GEMM on wgmma (wg_gemm_kernel) over "k8 planes" (see conv_tc.cu): for each
// group of 8 channels a hi and a lo plane of [rows][8] fp16, one row per group column (8 audio samples).  A GEMM's K
// is a list of segments, each a run of 64-channel chunks of some planes read at a row shift, so the dilated k=3
// convolution of a WN layer and its conditioning 1x1 convolution are ONE GEMM over
//     [h(t - d); h(t); h(t + d); spect(t)]      K = 3 * 256 + 640 = 1408, N = 512
// whose epilogue applies tanh * sigmoid (glow.py:34-40) -- cond_layer(spect) (glow.py:159) is never materialised.
//
// Rows: sequence b's group column t is row kGuard + b * span + t, span = 32 T_mel + kGuard; the kGuard = 128 rows
// after every sequence (and before the first) are zero, which is the zero padding of the largest dilation (128).
// With lengths, the rows t >= 32 len_b are kept zero as well, so a row sees exactly the padding it has alone.
//
//   upsample (glow.py:252-258)   ConvTranspose1d(80, 80, 1024, stride 256) as one GEMM over frames: output column
//                                n = mel * 256 + phase, K = 4 taps (frames F - j) x 80 mels; the epilogue writes the
//                                trimmed, unfolded (640, 32 T_mel) conditioning planes directly.
//   per flow (glow.py:271-290)   start (CUDA cores) -> 8 x [gate GEMM, res/skip GEMM] -> flow tail (CUDA cores, one
//                                thread per column): end, (a1 - b) / exp(s), the inverse 1x1 conv, the early noise,
//                                and the next flow's start (or the final (B, 8 L) interleave, glow.py:292).
//
// Tiers: fp32-grade = hi*hi + lo*hi + hi*lo (3 MMAs per K step); fp16 = hi*hi only, lo planes neither read nor written.
#include <math.h>
#include <stdlib.h>
#include <algorithm>
#include <string.h>

#include "conv_tc.h"
#include "waveglow.h"
#include "wg_gemm.cuh"

struct T2WaveGlow {
  int fp16;
  uint8_t* up_img = nullptr; float* up_bias = nullptr;
  uint8_t* gate_img[12][8] = {}; float* gate_bias = nullptr;     // (12, 8, 512), packed column order
  uint8_t* rs_img[12][8] = {};   float* rs_bias = nullptr;       // (12, 8, 512)
  struct t2_flow_w* flows = nullptr;
  float* tmp = nullptr;                                         // fp32 staging of the matrices being packed
};

struct t2_flow_w {                 // per flow, fp32, weight norm folded
  float end_w[8][256]; float end_b[8];
  float winv[8][8];
  float start_w[256][4]; float start_b[256];
};

namespace t2 {
namespace {

constexpr int kFlows = 12, kLayers = 8, kCond = 640, kGroup = 8;
#ifdef T2_SELFTEST
// waveglow_infer_window enqueues mel_to_planes, the upsample GEMM, the initial tail, then per flow 8 x (gate GEMM,
// res/skip GEMM) and a tail.
constexpr int kLaunches = 3 + kFlows * (2 * kLayers + 1);
// waveglow_state reads the workspace between two launches: waveglow_infer_window returns before launch g_stop_before
// (counted from 0; -1: never).  The product build has no stop points.
int g_stop_before = -1, g_launched = 0;
#define WG_STOP_POINT() do { if (g_launched++ == g_stop_before) return T2_OK; } while (0)
#else
#define WG_STOP_POINT() do {} while (0)
#endif
constexpr int kGuard = 128;                 // zero rows around each sequence in the column domain (max dilation)
constexpr int kFGuard = 4;                  // frame domain: 4 zero frames after each sequence (3 taps look back)
constexpr int kUpK = 4 * 128;               // upsample K: 4 taps x 80 mels padded to 128
// Receptive field of infer, in group columns (32 per frame).  One flow: the WN's dilated k = 3 layers reach
// +-(1 + 2 + ... + 128) = +-255 columns; start, end, the coupling, the inverse 1x1 conv and the noise act per column.
// Twelve flows: +-3060.  The upsample gives a column of frame f the frames f-3 ... f.  So the audio of frames [t0, t1)
// is fixed by the frames [t0 - 96 - 3, t1 + 96).
constexpr int kFlowReach = 255;
constexpr int kUpLook = 3;
constexpr int kHaloRight = (kFlows * kFlowReach + 31) / 32;   // 96 frames
constexpr int kHaloLeft = kHaloRight + kUpLook;                // 99 frames

// ---- Philox normal draws ----------------------------------------------------------------------------
// z(b, c, t): Philox4x32-10 with counter (t, b, c, kNoiseTag) and key (seed lo, seed hi); Box-Muller on the first
// two output words: u1 = ((o0 >> 8) + 1) 2^-24 in (0, 1], u2 = (o1 >> 8) 2^-24, z = sqrt(-2 ln u1) cos(2 pi u2).
constexpr uint32_t kNoiseTag = 0x3c6ef372u;
__device__ __forceinline__ float philox_normal(uint64_t seed, int b, int c, int t) {
  uint32_t o[4];
  philox4x32_10((uint32_t)t, (uint32_t)b, (uint32_t)c, kNoiseTag, (uint32_t)seed, (uint32_t)(seed >> 32), o);
  const float u1 = (float)((o[0] >> 8) + 1u) * (1.0f / 16777216.0f);
  const float u2 = (float)(o[1] >> 8) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cosf(6.28318530717958647692f * u2);
}

struct TailParams {
  const t2_flow_w* fw;
  int k;                 // flow whose WN just ran (-1: none, draw the initial noise)
  int next;              // flow whose start runs next, -1: write the audio
  int B, span, T; const int32_t* len; long n_rows;
  float sigma; const float* z; uint64_t seed;
  const float* skip; float* aud;
  __half* h; long h_rows;
  void* audio; int io_half;
};
// The window's fields are a separate kernel argument: added to TailParams they changed the tail kernel's code (39 -> 32
// registers, more constant-bank reloads) and made it about 30 % slower on the full sequence.
struct TailRange {
  int lo, hi;            // rows with t in [lo, hi) are computed; with next = -1 they are the audio written
  int col0; long z_stride;   // noise of window column t: absolute column col0 + t; rows of an injected z
};

__device__ __forceinline__ int n_rem_of(int k) { return 8 - 2 * (k / 4); }   // 4 (k >= 8), 6 (k >= 4), 8

template <int PASSES>
__global__ void __launch_bounds__(128) flow_tail_kernel(const TailParams p, const TailRange w) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.n_rows) return;
  const int b = (int)(q / p.span), t = (int)(q - (long)b * p.span);
  const bool data = b < p.B && t < p.T;
  if (data && (t < w.lo || t >= w.hi)) return;     // not needed by what follows
  const bool valid = data && (p.len == nullptr || t < p.len[b] * 32);
  auto noise = [&](int c) -> float {
    if (!valid) return 0.f;
    const int ta = w.col0 + t;
    return p.sigma * (p.z ? p.z[((long)b * kGroup + c) * w.z_stride + ta] : philox_normal(p.seed, b, c, ta));
  };
  float a[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = 0.f;
  if (p.k < 0) {                                   // glow.py:260-269
#pragma unroll
    for (int c = 0; c < 4; ++c) a[c] = noise(c);
  } else if (valid) {
    const t2_flow_w& f = p.fw[p.k];
    const int nr = n_rem_of(p.k), nh = nr / 2;
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c < nr) a[c] = p.aud[q * 8 + c];
    // end (glow.py:175) over the accumulated skip output
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.f;
    const float* sk = p.skip + q * kC;
    for (int c = 0; c < kC; c += 4) {
      const float4 s4 = *reinterpret_cast<const float4*>(sk + c);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < 2 * nh) {
          const float4 w4 = *reinterpret_cast<const float4*>(&f.end_w[j][c]);
          o[j] = fmaf(w4.x, s4.x, fmaf(w4.y, s4.y, fmaf(w4.z, s4.z, fmaf(w4.w, s4.w, o[j]))));
        }
    }
    // audio_1 = (audio_1 - b) / exp(s)  (glow.py:278-281)
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i < nh) a[nh + i] = (a[nh + i] - (o[i] + f.end_b[i])) / expf(o[nh + i] + f.end_b[nh + i]);
    // inverse 1x1 convolution (glow.py:283, 91-96)
    float na[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) if (r < nr && c < nr) acc = fmaf(f.winv[r][c], a[c], acc);
      na[r] = acc;
    }
    if (p.k % 4 == 0 && p.k > 0) {                 // early output: cat(sigma * z, audio)  (glow.py:285-290)
      const int zc = p.k == 8 ? 4 : 6;
#pragma unroll
      for (int r = 7; r >= 2; --r) a[r] = na[r - 2];
      a[0] = noise(zc); a[1] = noise(zc + 1);
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) a[r] = na[r];
    }
  }
  if (p.next >= 0) {
#pragma unroll
    for (int c = 0; c < 8; ++c) p.aud[q * 8 + c] = valid ? a[c] : 0.f;
    // start of the next flow (glow.py:155): h = W_start a[:n_half] + b
    const t2_flow_w& f = p.fw[p.next];
    const int nh = n_rem_of(p.next) / 2;
    for (int g = 0; g < kC / 8; ++g) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = g * 8 + i;
        float acc = f.start_b[c];
#pragma unroll
        for (int j = 0; j < 4; ++j) if (j < nh) acc = fmaf(f.start_w[c][j], a[j], acc);
        v[i] = valid ? acc : 0.f;
      }
      store8<PASSES>(p.h, p.h_rows, g, kGuard + q, v);
    }
  } else if (data) {                               // glow.py:292: audio[b, 8 (t - lo) + c], rows of 8 (hi - lo)
    const long o0 = (long)b * 8 * (w.hi - w.lo) + 8L * (t - w.lo);
    if (p.io_half) {
      __half* out = reinterpret_cast<__half*>(p.audio) + o0;
#pragma unroll
      for (int c = 0; c < 8; ++c) out[c] = __float2half_rn(valid ? a[c] : 0.f);
    } else {
      float* out = reinterpret_cast<float*>(p.audio) + o0;
#pragma unroll
      for (int c = 0; c < 8; ++c) out[c] = valid ? a[c] : 0.f;
    }
  }
}

// mel (B, 80, T) -> frame-domain planes (16 groups, channels >= 80 zero); frames >= len zero; every row written
__global__ void mel_to_planes_kernel(const void* __restrict__ mel, int io_half, int B, int T, const int32_t* __restrict__ len,
                                     __half* __restrict__ planes, long rows, int passes) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y;
  if (row >= rows) return;
  const long q = row - kFGuard;
  const int span = T + kFGuard;
  int b = -1, f = -1;
  if (q >= 0) { b = (int)(q / span); f = (int)(q - (long)b * span); }
  const bool valid = b >= 0 && b < B && f < T && (len == nullptr || f < len[b]);
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    float x = 0.f;
    if (valid && c < 80) {
      const long idx = ((long)b * 80 + c) * T + f;
      x = io_half ? __half2float(reinterpret_cast<const __half*>(mel)[idx]) : reinterpret_cast<const float*>(mel)[idx];
    }
    v[i] = x;
  }
  if (passes == 3) store8<3>(planes, rows, g, row, v);
  else store8<1>(planes, rows, g, row, v);
}

// ---- weight packing ----------------------------------------------------------------------------------
__device__ __forceinline__ float ldw(const void* p, long i, int half) {
  return half ? __half2float(reinterpret_cast<const __half*>(p)[i]) : reinterpret_cast<const float*>(p)[i];
}
// g / ||v|| of row n of a weight-normed tensor (1 when g is null: the weight is plain); 256 threads
__device__ float wn_scale(const void* v, const void* g, long n, int per_row, int half) {
  __shared__ float red[8];
  __shared__ float res;
  if (g == nullptr) return 1.f;
  float ss = 0.f;
  for (int i = threadIdx.x; i < per_row; i += blockDim.x) { const float x = ldw(v, n * per_row + i, half); ss += x * x; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    res = ldw(g, n, half) / sqrtf(tot);
  }
  __syncthreads();
  const float r = res;
  __syncthreads();
  return r;
}

// gate GEMM weight [512][1408]: packed row nn = tile * 256 + h * 128 + r is source row h * 256 + tile * 128 + r
// (tanh rows, then the matching sigmoid rows); K = [in_layer tap 0 | tap 1 | tap 2 | cond slice]
__global__ void build_gate_kernel(const void* in_b, const void* in_g, const void* in_v, const void* cond_b,
                                  const void* cond_g, const void* cond_v, int layer, int half, float* w, float* bias) {
  const int nn = blockIdx.x;
  const int n = ((nn >> 7) & 1) * 256 + (nn >> 8) * 128 + (nn & 127);
  const long nc = (long)layer * 512 + n;
  const float si = wn_scale(in_v, in_g, n, kC * 3, half);
  const float sc = wn_scale(cond_v, cond_g, nc, kCond, half);
  for (int k = threadIdx.x; k < 3 * kC + kCond; k += blockDim.x) {
    float x;
    if (k < 3 * kC) { const int tap = k / kC, ci = k % kC; x = ldw(in_v, ((long)n * kC + ci) * 3 + tap, half) * si; }
    else x = ldw(cond_v, nc * kCond + (k - 3 * kC), half) * sc;
    w[(long)nn * (3 * kC + kCond) + k] = x;
  }
  if (threadIdx.x == 0) bias[nn] = ldw(in_b, n, half) + ldw(cond_b, nc, half);
}

__global__ void build_rs_kernel(const void* rs_b, const void* rs_g, const void* rs_v, int half, float* w, float* bias) {
  const int n = blockIdx.x;
  const float s = wn_scale(rs_v, rs_g, n, kC, half);
  for (int k = threadIdx.x; k < kC; k += blockDim.x) w[(long)n * kC + k] = ldw(rs_v, (long)n * kC + k, half) * s;
  if (threadIdx.x == 0) bias[n] = ldw(rs_b, n, half);
}

// upsample as a GEMM: row n = o * 256 + phase, k = tap * 128 + i:  W[i][o][phase + 256 tap]
__global__ void build_up_kernel(const void* up_w, const void* up_b, int half, float* w, float* bias) {
  const int n = blockIdx.x, o = n >> 8, ph = n & 255;
  for (int k = threadIdx.x; k < kUpK; k += blockDim.x) {
    const int tap = k >> 7, i = k & 127;
    w[(long)n * kUpK + k] = i < 80 ? ldw(up_w, ((long)i * 80 + o) * 1024 + ph + 256 * tap, half) : 0.f;
  }
  if (threadIdx.x == 0 && ph == 0) bias[o] = ldw(up_b, o, half);
}

// start / end / inverse W of one flow; W^-1 by Gauss-Jordan with partial pivoting in double (once, at pack time)
__global__ void build_flow_kernel(const void* st_b, const void* st_g, const void* st_v, const void* end_w, const void* end_b,
                                  const float* convinv, int nr, int half, t2_flow_w* f) {
  const int nh = nr / 2;
  for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) {
    const int j = i / 256, c = i % 256;
    f->end_w[j][c] = j < nr ? ldw(end_w, (long)j * kC + c, half) : 0.f;
  }
  if (threadIdx.x < 8) f->end_b[threadIdx.x] = threadIdx.x < nr ? ldw(end_b, threadIdx.x, half) : 0.f;
  for (int c = 0; c < kC; ++c) {
    const float s = wn_scale(st_v, st_g, c, nh, half);
    if (threadIdx.x < 4) f->start_w[c][threadIdx.x] = threadIdx.x < nh ? ldw(st_v, (long)c * nh + threadIdx.x, half) * s : 0.f;
    if (threadIdx.x == 0) f->start_b[c] = ldw(st_b, c, half);
  }
  if (threadIdx.x == 0) {
    double m[8][16];
    for (int r = 0; r < nr; ++r)
      for (int c = 0; c < 2 * nr; ++c) m[r][c] = c < nr ? (double)convinv[r * nr + c] : (c - nr == r ? 1.0 : 0.0);
    for (int c = 0; c < nr; ++c) {
      int piv = c;
      for (int r = c + 1; r < nr; ++r) if (fabs(m[r][c]) > fabs(m[piv][c])) piv = r;
      for (int j = 0; j < 2 * nr; ++j) { const double x = m[c][j]; m[c][j] = m[piv][j]; m[piv][j] = x; }
      const double d = m[c][c];
      for (int j = 0; j < 2 * nr; ++j) m[c][j] /= d;
      for (int r = 0; r < nr; ++r)
        if (r != c) { const double e = m[r][c]; for (int j = 0; j < 2 * nr; ++j) m[r][j] -= e * m[c][j]; }
    }
    for (int r = 0; r < 8; ++r)
      for (int c = 0; c < 8; ++c) f->winv[r][c] = (r < nr && c < nr) ? (float)m[r][nr + c] : 0.f;
  }
}

// weight table indices (state_dict order): upsample (2), WN.k (56 each), convinv.k
constexpr int kWUpW = 0, kWUpB = 1;
constexpr int wn_base(int k) { return 2 + 56 * k; }
constexpr int kWConvinv = 2 + 56 * kFlows;
static_assert(kWConvinv + kFlows == T2_WAVEGLOW_NUM_WEIGHTS, "waveglow weight table");

int check_weights(const void* const* w, int n) {
  if (n != T2_WAVEGLOW_NUM_WEIGHTS) return fail(T2_ERR_INVALID, "waveglow: expected %d weight pointers, got %d", T2_WAVEGLOW_NUM_WEIGHTS, n);
  for (int i = 0; i < n; ++i) {
    const int o = (i - 2) % 56;            // weight_g entries may be null (plain weights after remove_weightnorm)
    const bool g_entry = i >= 2 && i < kWConvinv && ((o < 51 && o % 3 == 1) || o == 54);
    if (w[i] == nullptr && !g_entry) return fail(T2_ERR_INVALID, "waveglow: weight %d is null", i);
  }
  return T2_OK;
}

struct WsLayout {
  __half* x; long x_rows;
  __half* spect; __half* h; __half* acts; long rows;
  float* skip; float* aud;
};
struct Dims { int L, span, ntm, spanf, ntf; };
Dims dims_of(int B, int T) {
  Dims d;
  d.L = 32 * T; d.span = d.L + kGuard;
  d.ntm = (int)(((long)B * d.span + kTile - 1) / kTile);
  d.spanf = T + kFGuard;
  d.ntf = (int)(((long)B * d.spanf + kTile - 1) / kTile);
  return d;
}
void ws_layout(Carve& c, int B, int T, WsLayout* o) {
  const Dims d = dims_of(B, T);
  o->x_rows = kFGuard + (long)d.ntf * kTile;
  o->rows = kGuard + (long)d.ntm * kTile + kGuard;
  o->x = c.take<__half>((size_t)16 * 2 * o->x_rows * 8, 1024);
  o->spect = c.take<__half>((size_t)80 * 2 * o->rows * 8, 1024);
  o->h = c.take<__half>((size_t)32 * 2 * o->rows * 8, 1024);
  o->acts = c.take<__half>((size_t)32 * 2 * o->rows * 8, 1024);
  o->skip = c.take<float>((size_t)d.ntm * kTile * kC, 1024);
  o->aud = c.take<float>((size_t)d.ntm * kTile * 8, 1024);
}

#ifdef T2_SELFTEST
// planes -> fp32 rows (n_rows, 8 groups): tile row q is plane row kGuard + q; hi + lo in the fp32 tier, hi in the fp16 tier
__global__ void unpack_planes_kernel(const __half* __restrict__ planes, long rows, int passes, long n_rows,
                                     float* __restrict__ out) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y, groups = gridDim.y;
  if (q >= n_rows) return;
  float v[8];
  if (passes == 3) load8<3>(planes, rows, g, kGuard + q, v);
  else load8<1>(planes, rows, g, kGuard + q, v);
#pragma unroll
  for (int i = 0; i < 8; ++i) out[(q * groups + g) * 8 + i] = v[i];
}
#endif

}  // namespace

// ---- host API -----------------------------------------------------------------------------------------
static int pack(T2WaveGlow* m, const void* const* w, cudaStream_t s) {
  const int half = m->fp16;
  build_up_kernel<<<80 * 256, 256, 0, s>>>(w[kWUpW], w[kWUpB], half, m->tmp, m->up_bias);
  T2_LAUNCH_CHECK();
  T2_TRY(tc_pack_weights(m->tmp, 80 * 256, kUpK, 1, kNT, m->up_img, s));
  for (int k = 0; k < kFlows; ++k) {
    const int base = wn_base(k);
    const int nr = k >= 8 ? 4 : (k >= 4 ? 6 : 8);
    for (int l = 0; l < kLayers; ++l) {
      const int in = base + 3 * l, rs = base + 24 + 3 * l;
      float* gb = m->gate_bias + ((size_t)k * kLayers + l) * 512;
      build_gate_kernel<<<512, 256, 0, s>>>(w[in], w[in + 1], w[in + 2], w[base + 53], w[base + 54], w[base + 55], l, half,
                                             m->tmp, gb);
      T2_LAUNCH_CHECK();
      T2_TRY(tc_pack_weights(m->tmp, 512, 3 * kC + kCond, 1, kNT, m->gate_img[k][l], s));
      const int nrs = l < kLayers - 1 ? 512 : 256;
      float* rb = m->rs_bias + ((size_t)k * kLayers + l) * 512;
      build_rs_kernel<<<nrs, 256, 0, s>>>(w[rs], w[rs + 1], w[rs + 2], half, m->tmp, rb);
      T2_LAUNCH_CHECK();
      T2_TRY(tc_pack_weights(m->tmp, nrs, kC, 1, kNT, m->rs_img[k][l], s));
    }
    build_flow_kernel<<<1, 256, 0, s>>>(w[base + 48], w[base + 49], w[base + 50], w[base + 51], w[base + 52],
                                        reinterpret_cast<const float*>(w[kWConvinv + k]), nr, half, m->flows + k);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

int waveglow_create(T2WaveGlow** out, const T2WaveGlowConfig* c, const void* const* w, int n, cudaStream_t s) {
  if (!out || !c || !w) return fail(T2_ERR_INVALID, "waveglow: null argument");
  const bool ok = c->n_mel_channels == 80 && c->n_flows == kFlows && c->n_group == kGroup && c->n_early_every == 4 &&
                  c->n_early_size == 2 && c->wn_n_layers == kLayers && c->wn_kernel_size == 3 && c->wn_n_channels == kC &&
                  (c->fp16 == 0 || c->fp16 == 1);
  if (!ok)
    return fail(T2_ERR_UNSUPPORTED, "waveglow: configuration differs from the published one the sm_90a kernels are built for "
                                    "(n_mel 80, 12 flows, group 8, early 4 / 2, WN 8 layers x 256 channels, kernel 3)");
  T2_TRY(check_weights(w, n));
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) return fail(T2_ERR_UNSUPPORTED, "libt2b200 is built for sm_90a only (device is sm_%d%d)", p.major, p.minor);
  T2WaveGlow* m = new T2WaveGlow();
  m->fp16 = c->fp16;
  int r = T2_OK;
  if (cudaMalloc((void**)&m->up_bias, 80 * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->gate_bias, (size_t)kFlows * kLayers * 512 * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->rs_bias, (size_t)kFlows * kLayers * 512 * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->flows, kFlows * sizeof(t2_flow_w)) != cudaSuccess ||
      cudaMalloc((void**)&m->tmp, (size_t)80 * 256 * kUpK * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->up_img, tc_weights_bytes(80 * 256, kUpK, 1, kNT)) != cudaSuccess)
    r = fail(T2_ERR_CUDA, "waveglow: out of device memory for the packed weights");
  for (int k = 0; k < kFlows; ++k)
    for (int l = 0; l < kLayers && r == T2_OK; ++l)
      if (cudaMalloc((void**)&m->gate_img[k][l], tc_weights_bytes(512, 3 * kC + kCond, 1, kNT)) != cudaSuccess ||
          cudaMalloc((void**)&m->rs_img[k][l], tc_weights_bytes(l < kLayers - 1 ? 512 : 256, kC, 1, kNT)) != cudaSuccess)
        r = fail(T2_ERR_CUDA, "waveglow: out of device memory for the packed weights");
  if (r == T2_OK) r = pack(m, w, s);
  if (r != T2_OK) { waveglow_destroy(m); return r; }
  *out = m;
  return T2_OK;
}

int waveglow_refresh(T2WaveGlow* m, const void* const* w, int n, cudaStream_t s) {
  if (!m || !w) return fail(T2_ERR_INVALID, "waveglow: null argument");
  T2_TRY(check_weights(w, n));
  return pack(m, w, s);
}

int waveglow_destroy(T2WaveGlow* m) {
  if (!m) return T2_OK;
  cudaFree(m->up_img); cudaFree(m->up_bias); cudaFree(m->gate_bias); cudaFree(m->rs_bias); cudaFree(m->flows); cudaFree(m->tmp);
  for (int k = 0; k < kFlows; ++k)
    for (int l = 0; l < kLayers; ++l) { cudaFree(m->gate_img[k][l]); cudaFree(m->rs_img[k][l]); }
  delete m;
  return T2_OK;
}

size_t waveglow_ws_bytes(int B, int T) {
  Carve c(nullptr, 1024);
  WsLayout o;
  ws_layout(c, B, T, &o);
  return c.bytes();
}

void waveglow_window_halo(int* left, int* right) {
  if (left) *left = kHaloLeft;
  if (right) *right = kHaloRight;
}

int waveglow_infer(T2WaveGlow* m, const T2WaveGlowArgs* a, cudaStream_t s) {
  if (!a) return fail(T2_ERR_INVALID, "waveglow: null argument");
  T2WaveGlowWindowArgs w;
  memset(&w, 0, sizeof(w));
  w.wg = *a;
  w.frame0 = 0; w.out0 = 0; w.out1 = a->T_mel; w.z_frames = a->T_mel; w.at_end = 1;
  return waveglow_infer_window(m, &w, s);
}

int waveglow_infer_window(T2WaveGlow* m, const T2WaveGlowWindowArgs* wa, cudaStream_t s) {
  if (!m || !wa || !wa->wg.mel || !wa->wg.audio || !wa->wg.ws) return fail(T2_ERR_INVALID, "waveglow: null argument");
  const T2WaveGlowArgs* a = &wa->wg;
  if (a->B <= 0 || a->T_mel <= 0) return fail(T2_ERR_INVALID, "waveglow: empty input (B=%d, T_mel=%d)", a->B, a->T_mel);
  if ((long)a->B * (32L * a->T_mel + kGuard) > (1L << 30) || 32L * ((long)wa->frame0 + a->T_mel) > (1L << 30))
    return fail(T2_ERR_INVALID, "waveglow: input too large");
  const int frame0 = wa->frame0, out0 = wa->out0, out1 = wa->out1;
  if (frame0 < 0 || out0 < 0 || out1 <= out0 || out1 > a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: output frames [%d, %d) are not a non-empty range of the window's %d "
                "frames (frame0 %d)", out0, out1, a->T_mel, frame0);
  if (frame0 > 0 && out0 < kHaloLeft)
    return fail(T2_ERR_INVALID, "waveglow window: output frames start %d frames after a window start that is not the "
                "sequence's start; the left halo is %d frames", out0, kHaloLeft);
  if (!wa->at_end && out1 + kHaloRight > a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: output frames end %d frames before a window end that is not the "
                "sequence's end; the right halo is %d frames", a->T_mel - out1, kHaloRight);
  if (a->z && wa->z_frames < frame0 + a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: z holds %d frames, the window ends at frame %d", wa->z_frames,
                frame0 + a->T_mel);
  if (a->ws_bytes < waveglow_ws_bytes(a->B, a->T_mel)) return fail(T2_ERR_WORKSPACE, "waveglow workspace too small");
  const int B = a->B, T = a->T_mel, fp16 = m->fp16, passes = fp16 ? 1 : 3;
  const Dims d = dims_of(B, T);
  Carve c(a->ws, 1024);
  WsLayout o;
  ws_layout(c, B, T, &o);
  // Guard rows must read as zero: they are cleared here and only ever rewritten with zeros.  With per-flow ranges
  // (below) the rows a flow does not need are not rewritten and may hold stale values from earlier flows or calls
  // (skip and aud are not cleared at all); that is safe because no needed row reads an unneeded one.
  T2_CUDA(cudaMemsetAsync(o.spect, 0, (size_t)80 * 2 * o.rows * 16, s));
  T2_CUDA(cudaMemsetAsync(o.h, 0, (size_t)32 * 2 * o.rows * 16, s));
  T2_CUDA(cudaMemsetAsync(o.acts, 0, (size_t)32 * 2 * o.rows * 16, s));
  WG_STOP_POINT();
  mel_to_planes_kernel<<<dim3((unsigned)((o.x_rows + 127) / 128), 16), 128, 0, s>>>(a->mel, a->io_half, B, T, a->lengths,
                                                                                  o.x, o.x_rows, passes);
  T2_LAUNCH_CHECK();
  // upsample + trim + unfold (glow.py:252-258)
  GemmParams u;
  memset(&u, 0, sizeof(u));
  for (int j = 0; j < 4; ++j) u.seg[j] = Seg{o.x, o.x_rows, -j, 2};
  u.nseg = 4; u.nchunks = 8; u.row0 = kFGuard; u.wimg = m->up_img; u.n_tiles_m = d.ntf;
  u.B = B; u.span = d.spanf; u.T = T; u.lo = 0; u.hi = T; u.bias = m->up_bias;
  u.out = o.spect; u.out_rows = o.rows; u.out_row0 = kGuard; u.col_span = d.span;
  WG_STOP_POINT();
  T2_TRY(gemm<EPI_UPSAMPLE>(u, 80, fp16, s));

  // Per-flow column ranges.  The audio columns [32 out0, 32 out1) need the output of the flow that runs with n flows
  // still to follow over those columns widened by n * kFlowReach; that flow's WN layers run over one reach more.
  // Everything is clipped to the window: at a sequence edge the zero padding is the sequence's own.
  auto widen = [&](int n, int* lo, int* hi) {
    *lo = (int)std::max(0L, 32L * out0 - (long)kFlowReach * n);
    *hi = (int)std::min((long)d.L, 32L * out1 + (long)kFlowReach * n);
  };
  TailParams tp;
  memset(&tp, 0, sizeof(tp));
  tp.fw = m->flows; tp.B = B; tp.span = d.span; tp.T = d.L; tp.len = a->lengths; tp.n_rows = (long)d.ntm * kTile;
  tp.sigma = a->sigma; tp.z = a->z; tp.seed = a->seed;
  TailRange tr;
  tr.col0 = 32 * frame0; tr.z_stride = 32L * wa->z_frames;
  tp.skip = o.skip; tp.aud = o.aud; tp.h = o.h; tp.h_rows = o.rows;
  tp.audio = a->audio; tp.io_half = a->io_half;
  const unsigned tail_blocks = (unsigned)((tp.n_rows + 127) / 128);
  auto tail = [&](int k, int next) -> int {   // k flows follow this tail (k = 12: the initial draw)
    tp.k = k < kFlows ? k : -1; tp.next = next;
    widen(k, &tr.lo, &tr.hi);
    if (fp16) flow_tail_kernel<1><<<tail_blocks, 128, 0, s>>>(tp, tr);
    else flow_tail_kernel<3><<<tail_blocks, 128, 0, s>>>(tp, tr);
    T2_LAUNCH_CHECK();
    return T2_OK;
  };
  WG_STOP_POINT();
  T2_TRY(tail(kFlows, kFlows - 1));
  GemmParams g;
  memset(&g, 0, sizeof(g));
  g.row0 = kGuard; g.n_tiles_m = d.ntm; g.B = B; g.span = d.span; g.T = d.L; g.len = a->lengths; g.len_mul = 32;
  g.out_rows = o.rows; g.out_row0 = kGuard; g.skip = o.skip;
  for (int k = kFlows - 1; k >= 0; --k) {
    widen(k + 1, &g.lo, &g.hi);
    for (int l = 0; l < kLayers; ++l) {
      const int dil = 1 << l;
      // in_layer(audio) + cond_layer(spect)[slice] -> tanh * sigmoid  (glow.py:161-166)
      g.seg[0] = Seg{o.h, o.rows, -dil, 4}; g.seg[1] = Seg{o.h, o.rows, 0, 4}; g.seg[2] = Seg{o.h, o.rows, dil, 4};
      g.seg[3] = Seg{o.spect, o.rows, 0, 10};
      g.nseg = 4; g.nchunks = 22; g.wimg = m->gate_img[k][l]; g.bias = m->gate_bias + ((size_t)k * kLayers + l) * 512;
      g.out = o.acts;
      WG_STOP_POINT();
      T2_TRY(gemm<EPI_GATE>(g, 2, fp16, s));
      // res_skip_layers (glow.py:168-173)
      g.seg[0] = Seg{o.acts, o.rows, 0, 4};
      g.nseg = 1; g.nchunks = 4; g.wimg = m->rs_img[k][l]; g.bias = m->rs_bias + ((size_t)k * kLayers + l) * 512;
      g.out = o.h; g.first = l == 0; g.res_tiles = l < kLayers - 1 ? 1 : 0;
      WG_STOP_POINT();
      T2_TRY(gemm<EPI_RESSKIP>(g, l < kLayers - 1 ? 2 : 1, fp16, s));
    }
    WG_STOP_POINT();
    T2_TRY(tail(k, k > 0 ? k - 1 : -1));
  }
  return T2_OK;
}

#ifdef T2_SELFTEST
int waveglow_state(T2WaveGlow* m, const T2WaveGlowWindowArgs* wa, int n_launches, float* spect, float* hbuf, float* acts,
                   float* skip, float* aud, cudaStream_t s) {
  if (n_launches < 0 || n_launches > kLaunches)
    return fail(T2_ERR_INVALID, "waveglow state: n_launches %d is not in [0, %d]", n_launches, kLaunches);
  g_launched = 0; g_stop_before = n_launches;
  const int r = waveglow_infer_window(m, wa, s);
  g_stop_before = -1;
  T2_TRY(r);
  const int B = wa->wg.B, T = wa->wg.T_mel, passes = m->fp16 ? 1 : 3;
  Carve c(wa->wg.ws, 1024);
  WsLayout o;
  ws_layout(c, B, T, &o);
  const long n = (long)dims_of(B, T).ntm * kTile;
  const unsigned blocks = (unsigned)((n + 127) / 128);
  if (spect) unpack_planes_kernel<<<dim3(blocks, kCond / 8), 128, 0, s>>>(o.spect, o.rows, passes, n, spect);
  if (hbuf) unpack_planes_kernel<<<dim3(blocks, kC / 8), 128, 0, s>>>(o.h, o.rows, passes, n, hbuf);
  if (acts) unpack_planes_kernel<<<dim3(blocks, kC / 8), 128, 0, s>>>(o.acts, o.rows, passes, n, acts);
  T2_CUDA(cudaGetLastError());
  if (skip) T2_CUDA(cudaMemcpyAsync(skip, o.skip, (size_t)n * kC * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (aud) T2_CUDA(cudaMemcpyAsync(aud, o.aud, (size_t)n * 8 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return T2_OK;
}
#endif

}  // namespace t2
