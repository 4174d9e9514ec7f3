// WaveGlow inference (waveglow/glow.py:251-293, WaveGlow.infer) on sm_90a.
//
// Every dense product is one implicit GEMM on wgmma (wg_gemm_kernel) over "k8 planes" (see conv_tc.cu): for each
// group of 8 channels a hi and a lo plane of [rows][8] fp16, one row per group column (8 audio samples).  A GEMM's K
// is a list of segments, each a run of 64-channel chunks of some planes read at a row shift, so the dilated k=3
// convolution of a WN layer and its conditioning 1x1 convolution are ONE GEMM over
//     [h(t - d); h(t); h(t + d); spect(t)]      K = 3 C + 640, N = 2 C     (C = WN width: 128, 256, 384 or 512)
// whose epilogue applies tanh * sigmoid (glow.py:34-40) -- cond_layer(spect) (glow.py:159) is never materialised.
//
// Rows: sequence b's group column t is row guard + b * span + t, span = 32 T_mel + guard; the guard rows after every
// sequence (and before the first) are zero, which is the zero padding of the largest dilation (guard = 2^(n_layers-1),
// 128 for the published 8 layers).  With lengths, the rows t >= 32 len_b are kept zero as well, so a row sees exactly
// the padding it has alone.
//
//   upsample (glow.py:252-258)   ConvTranspose1d(80, 80, 1024, stride 256) as one GEMM over frames: output column
//                                n = mel * 256 + phase, K = 4 taps (frames F - j) x 80 mels; the epilogue writes the
//                                trimmed, unfolded (640, 32 T_mel) conditioning planes directly.
//   per flow (glow.py:271-290)   start (CUDA cores) -> n_layers x [gate GEMM, res/skip GEMM] -> flow tail (CUDA cores, one
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

namespace t2 {
namespace {

constexpr int kMaxFlows = 16, kMaxLayers = 10, kCond = 640, kGroup = 8;

// The shape of a supported configuration (waveglow_shape): every size below follows from it.
struct Shape {
  int C, layers, flows, early_every, early_size;
  constexpr int guard() const { return 1 << (layers - 1); }          // zero rows around each sequence: the largest dilation
  constexpr int reach() const { return (1 << layers) - 1; }          // one flow's WN reaches +-(1 + 2 + ... + guard) columns
  constexpr int halo_right() const { return (flows * reach() + 31) / 32; }
  constexpr int halo_left() const { return halo_right() + 3; }       // the upsample gives a column of frame f the frames f-3 ... f
  constexpr int n_rem(int k) const { return kGroup - early_size * (k / early_every); }   // channels flow k's coupling acts on
  constexpr int early(int k) const { return k > 0 && k % early_every == 0 ? early_size : 0; }
  constexpr int wn_entries() const { return 6 * layers + 8; }       // in_layers, res_skip_layers, start (3 each), end (2), cond (3)
  constexpr int wn_base(int k) const { return 2 + wn_entries() * k; }
  constexpr int convinv() const { return wn_base(flows); }
  constexpr int num_weights() const { return convinv() + flows; }
  constexpr int rs_rows(int l) const { return l < layers - 1 ? 2 * C : C; }
  constexpr int rs_tiles(int l) const { return (rs_rows(l) + 255) / 256; }   // the last layer's C rows padded to whole tiles
};

}  // namespace
}  // namespace t2

struct T2WaveGlow {
  int fp16;
  t2::Shape sh;
  uint8_t* up_img = nullptr; float* up_bias = nullptr;
  uint8_t* gate_img[16][10] = {}; float* gate_bias = nullptr;   // (flows, layers, 2C), packed column order
  uint8_t* rs_img[16][10] = {};   float* rs_bias = nullptr;     // (flows, layers, 2C)
  void* flows = nullptr;                                        // t2_flow_w<C>[flows]
  float* tmp = nullptr;                                         // fp32 staging of the matrices being packed
};

template <int C>
struct t2_flow_w {                 // per flow, fp32, weight norm folded
  float end_w[8][C]; float end_b[8];
  float winv[8][8];
  float start_w[C][4]; float start_b[C];
};
// the tail reads end_w as float4 from every flow of the array
static_assert(sizeof(t2_flow_w<128>) % 16 == 0 && sizeof(t2_flow_w<384>) % 16 == 0, "flow weights: float4 alignment");

namespace t2 {
namespace {

#ifdef T2_SELFTEST
// waveglow_infer_window enqueues mel_to_planes, the upsample GEMM, the initial tail, then per flow n_layers x (gate
// GEMM, res/skip GEMM) and a tail.
int launches_of(const Shape& sh) { return 3 + sh.flows * (2 * sh.layers + 1); }
// waveglow_state reads the workspace between two launches: waveglow_infer_window returns before launch g_stop_before
// (counted from 0; -1: never).  The product build has no stop points.
int g_stop_before = -1, g_launched = 0;
#define WG_STOP_POINT() do { if (g_launched++ == g_stop_before) return T2_OK; } while (0)
#else
#define WG_STOP_POINT() do {} while (0)
#endif
constexpr int kFGuard = 4;                  // frame domain: 4 zero frames after each sequence (3 taps look back)
constexpr int kUpK = 4 * 128;               // upsample K: 4 taps x 80 mels padded to 128
// Receptive field of infer, in group columns (32 per frame).  One flow: the WN's dilated k = 3 layers reach
// +-(2^n_layers - 1) columns (+-255 for 8 layers); start, end, the coupling, the inverse 1x1 conv and the noise act
// per column.  n_flows flows: +-n_flows (2^n_layers - 1) (+-3060 published).  The upsample gives a column of frame f
// the frames f-3 ... f.  So the audio of frames [t0, t1) is fixed by the frames [t0 - halo_right - 3, t1 + halo_right)
// (Shape::halo_left / halo_right; 99 and 96 frames published).

// ---- GEMM epilogues -------------------------------------------------------------------------------------
// gate: columns [0, 128) of the tile are the tanh inputs of channels nt*128 + c, [128, 256) their sigmoid inputs
// (the packed column order of build_gate_kernel); tanh * sigmoid goes to the acts planes
struct GateEpi : EpiDefaults {
  struct Params { const float* bias; __half* out; long out_rows, out_row0; };
  template <int PASSES, int NT, int NH>
  static __device__ __forceinline__ void apply(const Main& m, const Params& p, const float* row, int r, int half, long q,
                                               int b, int t, int nt, bool data, bool valid) {
    const float* bias = p.bias + nt * 256;
    for (int g = 0; g < 8; ++g) {
      const int c0 = half * 64 + g * 8;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xt = row[c0 + i] + bias[c0 + i], xs = row[128 + c0 + i] + bias[128 + c0 + i];
        v[i] = valid ? tanhf(xt) * (1.f / (1.f + expf(-xs))) : 0.f;
      }
      store8<PASSES>(p.out, p.out_rows, nt * 16 + (c0 >> 3), p.out_row0 + q, v);
    }
  }
};

// res/skip: output columns < res_cols are the residual half, added to the h planes `out`; the next skip_cols columns
// are the skip half, stored (first) or added to the fp32 skip rows; later columns are padding
struct ResSkipEpi : EpiDefaults {
  struct Params { const float* bias; __half* out; long out_rows, out_row0; float* skip; int first, res_cols, skip_cols; };
  template <int PASSES, int NT, int NH>
  static __device__ __forceinline__ void apply(const Main& m, const Params& p, const float* row, int r, int half, long q,
                                               int b, int t, int nt, bool data, bool valid) {
    // each thread's 128 columns lie wholly in the residual half or the skip half (the WN width is a multiple of 128)
    const int n0 = nt * 256 + half * 128;
    if (n0 < p.res_cols) {             // audio = audio + res_skip_acts[:, :C]  (glow.py:170)
      for (int g = 0; g < 16; ++g) {
        const int c0 = n0 + g * 8;
        float v[8];
        load8<PASSES>(p.out, p.out_rows, c0 >> 3, p.out_row0 + q, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = valid ? v[i] + (row[c0 - nt * 256 + i] + p.bias[c0 + i]) : 0.f;
        store8<PASSES>(p.out, p.out_rows, c0 >> 3, p.out_row0 + q, v);
      }
    } else if (n0 - p.res_cols < p.skip_cols) {   // output = output + res_skip_acts[:, C:]  (glow.py:171, 173)
      float* sk = p.skip + q * p.skip_cols + (n0 - p.res_cols);
      for (int c = 0; c < 128; c += 4) {
        float4 x = make_float4(row[half * 128 + c] + p.bias[n0 + c], row[half * 128 + c + 1] + p.bias[n0 + c + 1],
                               row[half * 128 + c + 2] + p.bias[n0 + c + 2], row[half * 128 + c + 3] + p.bias[n0 + c + 3]);
        if (!p.first) {
          const float4 o = *reinterpret_cast<const float4*>(sk + c);
          x.x += o.x; x.y += o.y; x.z += o.z; x.w += o.w;
        }
        *reinterpret_cast<float4*>(sk + c) = x;
      }
    }
  }
};

// upsample: column tile nt = mel channel, column = phase; frame row t writes the conditioning planes' group columns
// 32 t ... 32 t + 31 of sequence b (plane row out_row0 + b * col_span + column)
struct UpsampleEpi : EpiDefaults {
  struct Params { const float* bias; __half* out; long out_rows, out_row0; int col_span; };
  template <int PASSES, int NT, int NH>
  static __device__ __forceinline__ void apply(const Main& m, const Params& p, const float* row, int r, int half, long q,
                                               int b, int t, int nt, bool data, bool valid) {
    if (data) {
      const float bo = p.bias[nt];
      const long crow = p.out_row0 + (long)b * p.col_span + 32L * t + half * 16;
      for (int k = 0; k < 16; ++k) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = row[half * 128 + k * 8 + i] + bo;
        store8<PASSES>(p.out, p.out_rows, nt, crow + k, v);
      }
    }
  }
};

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

template <int C>
struct TailParams {
  const t2_flow_w<C>* fw;
  int k;                 // flow whose WN just ran (-1: none, draw the initial noise)
  int next;              // flow whose start runs next, -1: write the audio
  int B, span, T; const int32_t* len; long n_rows;
  float sigma; const float* z; uint64_t seed;
  const float* skip; float* aud;
  __half* h; long h_rows;       // h points at the planes' guard row: tile row q is row q of each plane
  void* audio; int io_half;
};
// The window's fields are a separate kernel argument: added to TailParams they changed the tail kernel's code (39 -> 32
// registers, more constant-bank reloads) and made it about 30 % slower on the full sequence.
struct TailRange {
  int lo, hi;            // rows with t in [lo, hi) are computed; with next = -1 they are the audio written
  int col0; long z_stride;   // noise of window column t: absolute column col0 + t; rows of an injected z
  // The flow schedule as launch arguments, so that every branch on it is uniform: channels flow k acts on (k < 0: the
  // channels of the initial draw), the early output after it (0: none) and the next flow's n_half.
  int nr, early, nh_next;
};

// a[r] = na[r - e] for r >= e (the channels before are the early noise's), e = 4 or 6; kept out of line so that the
// common 2-channel schedule compiles to the tail's straight-line code
__device__ __noinline__ void early_shift(const float* na, int e, float* a) {
#pragma unroll
  for (int r = 0; r < 8; ++r) a[r] = r >= 6 ? (e == 4 ? na[r - 4] : na[r - 6]) : (r >= 4 && e == 4 ? na[r - 4] : 0.f);
}

// SEEDED: row b draws its noise as a B = 1 call with seed row_seeds[b] does -- key row_seeds[b], row index 0.  A
// template parameter, so that the unseeded instantiation compiles to the code it had before row_seeds existed.
// C: the WN width.  The flow schedule (channels per flow, early outputs) comes with the range w.
template <int PASSES, bool SEEDED, int C>
__global__ void __launch_bounds__(128) flow_tail_kernel(const TailParams<C> p, const TailRange w,
                                                        const uint64_t* __restrict__ row_seeds) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.n_rows) return;
  const int b = (int)(q / p.span), t = (int)(q - (long)b * p.span);
  const bool data = b < p.B && t < p.T;
  if (data && (t < w.lo || t >= w.hi)) return;     // not needed by what follows
  const bool valid = data && (p.len == nullptr || t < p.len[b] * 32);
  const uint64_t seed = SEEDED && valid ? row_seeds[b] : p.seed;
  auto noise = [&](int c) -> float {
    if (!valid) return 0.f;
    const int ta = w.col0 + t;
    if (SEEDED) return p.sigma * philox_normal(seed, 0, c, ta);
    return p.sigma * (p.z ? p.z[((long)b * kGroup + c) * w.z_stride + ta] : philox_normal(p.seed, b, c, ta));
  };
  float a[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = 0.f;
  if (p.k < 0) {                                   // glow.py:260-269
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c < w.nr) a[c] = noise(c);
  } else if (valid) {
    const t2_flow_w<C>& f = p.fw[p.k];
    const int nr = w.nr, nh = nr / 2;
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c < nr) a[c] = p.aud[q * 8 + c];
    // end (glow.py:175) over the accumulated skip output
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.f;
    const float* sk = p.skip + q * C;
    for (int c = 0; c < C; c += 4) {
      const float4 s4 = *reinterpret_cast<const float4*>(sk + c);
      float4 w4[8];                                // every row's weights issued before the first use
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < 2 * nh) w4[j] = *reinterpret_cast<const float4*>(&f.end_w[j][c]);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < 2 * nh) o[j] = fmaf(w4[j].x, s4.x, fmaf(w4[j].y, s4.y, fmaf(w4[j].z, s4.z, fmaf(w4[j].w, s4.w, o[j]))));
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
    // early output: cat(sigma * z[nr, nr + e), audio)  (glow.py:285-290), e = 2, 4 or 6 channels
    const int e = w.early;
    if (e == 2) {
#pragma unroll
      for (int r = 7; r >= 2; --r) a[r] = na[r - 2];
      a[0] = noise(nr); a[1] = noise(nr + 1);
    } else if (e > 0) {
      early_shift(na, e, a);
#pragma unroll
      for (int r = 0; r < 6; ++r) if (r < e) a[r] = noise(nr + r);
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) a[r] = na[r];
    }
  }
  if (p.next >= 0) {
#pragma unroll
    for (int c = 0; c < 8; ++c) p.aud[q * 8 + c] = valid ? a[c] : 0.f;
    // start of the next flow (glow.py:155): h = W_start a[:n_half] + b
    const t2_flow_w<C>& f = p.fw[p.next];
    const int nh = w.nh_next;
    for (int g = 0; g < C / 8; ++g) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = g * 8 + i;
        float acc = f.start_b[c];
#pragma unroll
        for (int j = 0; j < 4; ++j) if (j < nh) acc = fmaf(f.start_w[c][j], a[j], acc);
        v[i] = valid ? acc : 0.f;
      }
      store8<PASSES>(p.h, p.h_rows, g, q, v);
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

// ---- weight packing ----------------------------------------------------------------------------------
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

// gate GEMM weight [2C][3C + 640]: packed row nn = tile * 256 + h * 128 + r is source row h * C + tile * 128 + r
// (tanh rows, then the matching sigmoid rows); K = [in_layer tap 0 | tap 1 | tap 2 | cond slice]
__global__ void build_gate_kernel(const void* in_b, const void* in_g, const void* in_v, const void* cond_b,
                                  const void* cond_g, const void* cond_v, int layer, int C, int half, float* w, float* bias) {
  const int nn = blockIdx.x;
  const int n = ((nn >> 7) & 1) * C + (nn >> 8) * 128 + (nn & 127);
  const long nc = (long)layer * 2 * C + n;
  const float si = wn_scale(in_v, in_g, n, C * 3, half);
  const float sc = wn_scale(cond_v, cond_g, nc, kCond, half);
  for (int k = threadIdx.x; k < 3 * C + kCond; k += blockDim.x) {
    float x;
    if (k < 3 * C) { const int tap = k / C, ci = k % C; x = ldw(in_v, ((long)n * C + ci) * 3 + tap, half) * si; }
    else x = ldw(cond_v, nc * kCond + (k - 3 * C), half) * sc;
    w[(long)nn * (3 * C + kCond) + k] = x;
  }
  if (threadIdx.x == 0) bias[nn] = ldw(in_b, n, half) + ldw(cond_b, nc, half);
}

// res/skip weight [gridDim.x][C]: rows n >= n_out (the padding of the last layer's C rows to whole tiles) are zero
__global__ void build_rs_kernel(const void* rs_b, const void* rs_g, const void* rs_v, int C, int n_out, int half, float* w,
                                float* bias) {
  const int n = blockIdx.x;
  if (n >= n_out) {
    for (int k = threadIdx.x; k < C; k += blockDim.x) w[(long)n * C + k] = 0.f;
    if (threadIdx.x == 0) bias[n] = 0.f;
    return;
  }
  const float s = wn_scale(rs_v, rs_g, n, C, half);
  for (int k = threadIdx.x; k < C; k += blockDim.x) w[(long)n * C + k] = ldw(rs_v, (long)n * C + k, half) * s;
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
template <int C>
__global__ void build_flow_kernel(const void* st_b, const void* st_g, const void* st_v, const void* end_w, const void* end_b,
                                  const float* convinv, int nr, int half, t2_flow_w<C>* f) {
  const int nh = nr / 2;
  for (int i = threadIdx.x; i < 8 * C; i += blockDim.x) {
    const int j = i / C, c = i % C;
    f->end_w[j][c] = j < nr ? ldw(end_w, (long)j * C + c, half) : 0.f;
  }
  if (threadIdx.x < 8) f->end_b[threadIdx.x] = threadIdx.x < nr ? ldw(end_b, threadIdx.x, half) : 0.f;
  for (int c = 0; c < C; ++c) {
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

// weight table indices (state_dict order): upsample (2), WN.k (Shape::wn_entries each), convinv.k
constexpr int kWUpW = 0, kWUpB = 1;
constexpr Shape kPublished{256, 8, 12, 4, 2};
static_assert(kPublished.num_weights() == T2_WAVEGLOW_NUM_WEIGHTS, "waveglow weight table");

// The supported configurations (see include/t2b200.h); 0 with *sh filled in, or a message for the first violation.
const char* waveglow_shape(const T2WaveGlowConfig* c, Shape* sh) {
  if (c->n_mel_channels != 80) return "n_mel_channels must be 80";
  if (c->n_group != kGroup) return "n_group must be 8";
  if (c->wn_kernel_size != 3) return "WN kernel_size must be 3";
  if (c->wn_n_channels < 128 || c->wn_n_channels > 512 || c->wn_n_channels % 128)
    return "WN n_channels must be 128, 256, 384 or 512";
  if (c->wn_n_layers < 1 || c->wn_n_layers > kMaxLayers) return "WN n_layers must be in [1, 10]";
  if (c->n_flows < 1 || c->n_flows > kMaxFlows) return "n_flows must be in [1, 16]";
  if (c->n_early_every < 1) return "n_early_every must be at least 1";
  if (c->n_early_size < 0 || c->n_early_size % 2) return "n_early_size must be even and not negative";
  if (c->fp16 != 0 && c->fp16 != 1) return "fp16 must be 0 or 1";
  *sh = Shape{c->wn_n_channels, c->wn_n_layers, c->n_flows, c->n_early_every, c->n_early_size};
  if (sh->n_rem(c->n_flows - 1) < 2) return "the early outputs leave fewer than 2 channels to the last flow";
  return nullptr;
}

int check_weights(const Shape& sh, const void* const* w, int n) {
  if (n != sh.num_weights()) return fail(T2_ERR_INVALID, "waveglow: expected %d weight pointers, got %d", sh.num_weights(), n);
  const int per = sh.wn_entries(), st = 6 * sh.layers;
  for (int i = 0; i < n; ++i) {
    const int o = (i - 2) % per;           // weight_g entries may be null (plain weights after remove_weightnorm)
    const bool g_entry = i >= 2 && i < sh.convinv() && ((o < st + 3 && o % 3 == 1) || o == st + 6);
    if (w[i] == nullptr && !g_entry) return fail(T2_ERR_INVALID, "waveglow: weight %d is null", i);
  }
  return T2_OK;
}

size_t flow_bytes(int C) {
  switch (C) {
    case 128: return sizeof(t2_flow_w<128>);
    case 256: return sizeof(t2_flow_w<256>);
    case 384: return sizeof(t2_flow_w<384>);
    default: return sizeof(t2_flow_w<512>);
  }
}

struct WsLayout {
  __half* x; long x_rows;
  __half* spect; __half* h; __half* acts; long rows;
  float* skip; float* aud;
};
struct Dims { int L, span, ntm, spanf, ntf; };
Dims dims_of(const Shape& sh, int B, int T) {
  Dims d;
  d.L = 32 * T; d.span = d.L + sh.guard();
  d.ntm = (int)(((long)B * d.span + kTile - 1) / kTile);
  d.spanf = T + kFGuard;
  d.ntf = (int)(((long)B * d.spanf + kTile - 1) / kTile);
  return d;
}
void ws_layout(Carve& c, const Shape& sh, int B, int T, WsLayout* o) {
  const Dims d = dims_of(sh, B, T);
  o->x_rows = kFGuard + (long)d.ntf * kTile;
  o->rows = sh.guard() + (long)d.ntm * kTile + sh.guard();
  o->x = c.take<__half>(planes_bytes(128, o->x_rows) / sizeof(__half), 1024);
  o->spect = c.take<__half>(planes_bytes(kCond, o->rows) / sizeof(__half), 1024);
  o->h = c.take<__half>(planes_bytes(sh.C, o->rows) / sizeof(__half), 1024);
  o->acts = c.take<__half>(planes_bytes(sh.C, o->rows) / sizeof(__half), 1024);
  o->skip = c.take<float>((size_t)d.ntm * kTile * sh.C, 1024);
  o->aud = c.take<float>((size_t)d.ntm * kTile * 8, 1024);
}

#ifdef T2_SELFTEST
// planes -> fp32 rows (n_rows, 8 groups): tile row q is plane row kGuard + q; hi + lo in the fp32 tier, hi in the fp16 tier
__global__ void unpack_planes_kernel(const __half* __restrict__ planes, long rows, int guard, int passes, long n_rows,
                                     float* __restrict__ out) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y, groups = gridDim.y;
  if (q >= n_rows) return;
  float v[8];
  if (passes == 3) load8<3>(planes, rows, g, guard + q, v);
  else load8<1>(planes, rows, g, guard + q, v);
#pragma unroll
  for (int i = 0; i < 8; ++i) out[(q * groups + g) * 8 + i] = v[i];
}
#endif

}  // namespace

// ---- host API -----------------------------------------------------------------------------------------
template <int C>
static void launch_build_flow(const void* const* w, int base, const Shape& sh, const float* convinv, int k, int half,
                              void* flows, cudaStream_t s) {
  const int st = base + 6 * sh.layers;
  build_flow_kernel<C><<<1, 256, 0, s>>>(w[st], w[st + 1], w[st + 2], w[st + 3], w[st + 4], convinv, sh.n_rem(k), half,
                                         reinterpret_cast<t2_flow_w<C>*>(flows) + k);
}

static int pack(T2WaveGlow* m, const void* const* w, cudaStream_t s) {
  const int half = m->fp16;
  const Shape& sh = m->sh;
  const int C = sh.C, L = sh.layers;
  build_up_kernel<<<80 * 256, 256, 0, s>>>(w[kWUpW], w[kWUpB], half, m->tmp, m->up_bias);
  T2_LAUNCH_CHECK();
  T2_TRY(tc_pack_weights(m->tmp, 80 * 256, kUpK, 1, kNT, m->up_img, s));
  for (int k = 0; k < sh.flows; ++k) {
    const int base = sh.wn_base(k), cond = base + 6 * L + 5;
    for (int l = 0; l < L; ++l) {
      const int in = base + 3 * l, rs = base + 3 * L + 3 * l;
      float* gb = m->gate_bias + ((size_t)k * L + l) * 2 * C;
      build_gate_kernel<<<2 * C, 256, 0, s>>>(w[in], w[in + 1], w[in + 2], w[cond], w[cond + 1], w[cond + 2], l, C, half,
                                               m->tmp, gb);
      T2_LAUNCH_CHECK();
      T2_TRY(tc_pack_weights(m->tmp, 2 * C, 3 * C + kCond, 1, kNT, m->gate_img[k][l], s));
      const int nrs = 256 * sh.rs_tiles(l);
      float* rb = m->rs_bias + ((size_t)k * L + l) * 2 * C;
      build_rs_kernel<<<nrs, 256, 0, s>>>(w[rs], w[rs + 1], w[rs + 2], C, sh.rs_rows(l), half, m->tmp, rb);
      T2_LAUNCH_CHECK();
      T2_TRY(tc_pack_weights(m->tmp, nrs, C, 1, kNT, m->rs_img[k][l], s));
    }
    const float* convinv = reinterpret_cast<const float*>(w[sh.convinv() + k]);
    switch (C) {
      case 128: launch_build_flow<128>(w, base, sh, convinv, k, half, m->flows, s); break;
      case 256: launch_build_flow<256>(w, base, sh, convinv, k, half, m->flows, s); break;
      case 384: launch_build_flow<384>(w, base, sh, convinv, k, half, m->flows, s); break;
      default: launch_build_flow<512>(w, base, sh, convinv, k, half, m->flows, s); break;
    }
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

int waveglow_num_weights(const T2WaveGlowConfig* c) {
  Shape sh;
  return c && waveglow_shape(c, &sh) == nullptr ? sh.num_weights() : 0;
}

int waveglow_window_halo_config(const T2WaveGlowConfig* c, int* left, int* right) {
  if (!c) return fail(T2_ERR_INVALID, "waveglow: null argument");
  Shape sh;
  if (const char* why = waveglow_shape(c, &sh)) return fail(T2_ERR_UNSUPPORTED, "waveglow: unsupported configuration: %s", why);
  if (left) *left = sh.halo_left();
  if (right) *right = sh.halo_right();
  return T2_OK;
}

int waveglow_create(T2WaveGlow** out, const T2WaveGlowConfig* c, const void* const* w, int n, cudaStream_t s) {
  if (!out || !c || !w) return fail(T2_ERR_INVALID, "waveglow: null argument");
  Shape sh;
  if (const char* why = waveglow_shape(c, &sh))
    return fail(T2_ERR_UNSUPPORTED, "waveglow: the sm_90a kernels do not support this configuration: %s (supported: "
                                    "n_mel 80, group 8, 1-16 flows, WN 1-10 layers x 128/256/384/512 channels, kernel 3)", why);
  T2_TRY(check_weights(sh, w, n));
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) return fail(T2_ERR_UNSUPPORTED, "libt2b200 is built for sm_90a only (device is sm_%d%d)", p.major, p.minor);
  T2WaveGlow* m = new T2WaveGlow();
  m->fp16 = c->fp16;
  m->sh = sh;
  const int C = sh.C, L = sh.layers;
  int r = T2_OK;
  if (cudaMalloc((void**)&m->up_bias, 80 * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->gate_bias, (size_t)sh.flows * L * 2 * C * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->rs_bias, (size_t)sh.flows * L * 2 * C * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&m->flows, sh.flows * flow_bytes(C)) != cudaSuccess ||
      cudaMalloc((void**)&m->tmp, (size_t)80 * 256 * kUpK * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->up_img, tc_weights_bytes(80 * 256, kUpK, 1, kNT)) != cudaSuccess)
    r = fail(T2_ERR_CUDA, "waveglow: out of device memory for the packed weights");
  for (int k = 0; k < sh.flows; ++k)
    for (int l = 0; l < L && r == T2_OK; ++l)
      if (cudaMalloc((void**)&m->gate_img[k][l], tc_weights_bytes(2 * C, 3 * C + kCond, 1, kNT)) != cudaSuccess ||
          cudaMalloc((void**)&m->rs_img[k][l], tc_weights_bytes(256 * sh.rs_tiles(l), C, 1, kNT)) != cudaSuccess)
        r = fail(T2_ERR_CUDA, "waveglow: out of device memory for the packed weights");
  if (r == T2_OK) r = pack(m, w, s);
  if (r != T2_OK) { waveglow_destroy(m); return r; }
  *out = m;
  return T2_OK;
}

int waveglow_refresh(T2WaveGlow* m, const void* const* w, int n, cudaStream_t s) {
  if (!m || !w) return fail(T2_ERR_INVALID, "waveglow: null argument");
  T2_TRY(check_weights(m->sh, w, n));
  return pack(m, w, s);
}

int waveglow_destroy(T2WaveGlow* m) {
  if (!m) return T2_OK;
  cudaFree(m->up_img); cudaFree(m->up_bias); cudaFree(m->gate_bias); cudaFree(m->rs_bias); cudaFree(m->flows); cudaFree(m->tmp);
  for (int k = 0; k < m->sh.flows; ++k)
    for (int l = 0; l < m->sh.layers; ++l) { cudaFree(m->gate_img[k][l]); cudaFree(m->rs_img[k][l]); }
  delete m;
  return T2_OK;
}

size_t waveglow_ws_bytes(const T2WaveGlow* m, int B, int T) {
  Carve c(nullptr, 1024);
  WsLayout o;
  ws_layout(c, m ? m->sh : kPublished, B, T, &o);
  return c.bytes();
}

void waveglow_window_halo(int* left, int* right) {
  if (left) *left = kPublished.halo_left();
  if (right) *right = kPublished.halo_right();
}

int waveglow_infer(T2WaveGlow* m, const T2WaveGlowArgs* a, cudaStream_t s) {
  if (!a) return fail(T2_ERR_INVALID, "waveglow: null argument");
  T2WaveGlowWindowArgs w;
  memset(&w, 0, sizeof(w));
  w.wg = *a;
  w.frame0 = 0; w.out0 = 0; w.out1 = a->T_mel; w.z_frames = a->T_mel; w.at_end = 1;
  return waveglow_infer_window(m, &w, s);
}

// The initial tail and the flows of an infer_window, for WN width C
template <int C, class Widen>
static int run_flows(T2WaveGlow* m, const T2WaveGlowWindowArgs* wa, const WsLayout& o, const Dims& d, Widen widen,
                     cudaStream_t s) {
  const T2WaveGlowArgs* a = &wa->wg;
  const Shape& sh = m->sh;
  const int B = a->B, fp16 = m->fp16, guard = sh.guard(), L = sh.layers, flows = sh.flows;
  TailParams<C> tp;
  memset(&tp, 0, sizeof(tp));
  tp.fw = reinterpret_cast<const t2_flow_w<C>*>(m->flows); tp.B = B; tp.span = d.span; tp.T = d.L; tp.len = a->lengths;
  tp.n_rows = (long)d.ntm * kTile;
  tp.sigma = a->sigma; tp.z = a->z; tp.seed = a->seed;
  TailRange tr;
  tr.col0 = 32 * wa->frame0; tr.z_stride = 32L * wa->z_frames;
  tp.skip = o.skip; tp.aud = o.aud; tp.h = o.h + (size_t)guard * 8; tp.h_rows = o.rows;
  tp.audio = a->audio; tp.io_half = a->io_half;
  const unsigned tail_blocks = (unsigned)((tp.n_rows + 127) / 128);
  auto tail = [&](int k, int next) -> int {   // k flows follow this tail (k = flows: the initial draw)
    tp.k = k < flows ? k : -1; tp.next = next;
    widen(k, &tr.lo, &tr.hi);
    tr.nr = sh.n_rem(k < flows ? k : flows - 1); tr.early = k < flows ? sh.early(k) : 0;
    tr.nh_next = next >= 0 ? sh.n_rem(next) / 2 : 0;
    const uint64_t* rs = a->row_seeds;
    if (fp16) {
      if (rs) flow_tail_kernel<1, true, C><<<tail_blocks, 128, 0, s>>>(tp, tr, rs);
      else flow_tail_kernel<1, false, C><<<tail_blocks, 128, 0, s>>>(tp, tr, nullptr);
    } else {
      if (rs) flow_tail_kernel<3, true, C><<<tail_blocks, 128, 0, s>>>(tp, tr, rs);
      else flow_tail_kernel<3, false, C><<<tail_blocks, 128, 0, s>>>(tp, tr, nullptr);
    }
    T2_LAUNCH_CHECK();
    return T2_OK;
  };
  WG_STOP_POINT();
  T2_TRY(tail(flows, flows - 1));
  Main g;
  memset(&g, 0, sizeof(g));
  g.row0 = guard; g.n_tiles_m = d.ntm; g.B = B; g.span = d.span; g.T = d.L; g.len = a->lengths; g.len_mul = 32;
  const int cc = C / 64;                     // 64-channel chunks of h and acts
  for (int k = flows - 1; k >= 0; --k) {
    widen(k + 1, &g.lo, &g.hi);
    for (int l = 0; l < L; ++l) {
      const int dil = 1 << l;
      // in_layer(audio) + cond_layer(spect)[slice] -> tanh * sigmoid  (glow.py:161-166)
      g.seg[0] = Seg{o.h, o.rows, -dil, cc}; g.seg[1] = Seg{o.h, o.rows, 0, cc}; g.seg[2] = Seg{o.h, o.rows, dil, cc};
      g.seg[3] = Seg{o.spect, o.rows, 0, 10};
      g.nseg = 4; g.nchunks = 3 * cc + 10; g.wimg = m->gate_img[k][l];
      const GateEpi::Params ge{m->gate_bias + ((size_t)k * L + l) * 2 * C, o.acts, o.rows, guard};
      WG_STOP_POINT();
      T2_TRY(gemm<GateEpi>(g, ge, C / 128, fp16, s));
      // res_skip_layers (glow.py:168-173)
      g.seg[0] = Seg{o.acts, o.rows, 0, cc};
      g.nseg = 1; g.nchunks = cc; g.wimg = m->rs_img[k][l];
      const ResSkipEpi::Params re{m->rs_bias + ((size_t)k * L + l) * 2 * C, o.h, o.rows, guard, o.skip, l == 0,
                                  l < L - 1 ? C : 0, C};
      WG_STOP_POINT();
      T2_TRY(gemm<ResSkipEpi>(g, re, sh.rs_tiles(l), fp16, s));
    }
    WG_STOP_POINT();
    T2_TRY(tail(k, k > 0 ? k - 1 : -1));
  }
  return T2_OK;
}

int waveglow_infer_window(T2WaveGlow* m, const T2WaveGlowWindowArgs* wa, cudaStream_t s) {
  if (!m || !wa || !wa->wg.mel || !wa->wg.audio || !wa->wg.ws) return fail(T2_ERR_INVALID, "waveglow: null argument");
  const T2WaveGlowArgs* a = &wa->wg;
  const Shape& sh = m->sh;
  const int guard = sh.guard(), halo_left = sh.halo_left(), halo_right = sh.halo_right(), reach = sh.reach();
  if (a->B <= 0 || a->T_mel <= 0) return fail(T2_ERR_INVALID, "waveglow: empty input (B=%d, T_mel=%d)", a->B, a->T_mel);
  if ((long)a->B * (32L * a->T_mel + guard) > (1L << 30) || 32L * ((long)wa->frame0 + a->T_mel) > (1L << 30))
    return fail(T2_ERR_INVALID, "waveglow: input too large");
  const int frame0 = wa->frame0, out0 = wa->out0, out1 = wa->out1;
  if (frame0 < 0 || out0 < 0 || out1 <= out0 || out1 > a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: output frames [%d, %d) are not a non-empty range of the window's %d "
                "frames (frame0 %d)", out0, out1, a->T_mel, frame0);
  if (frame0 > 0 && out0 < halo_left)
    return fail(T2_ERR_INVALID, "waveglow window: output frames start %d frames after a window start that is not the "
                "sequence's start; the left halo is %d frames", out0, halo_left);
  if (!wa->at_end && out1 + halo_right > a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: output frames end %d frames before a window end that is not the "
                "sequence's end; the right halo is %d frames", a->T_mel - out1, halo_right);
  if (a->z && a->row_seeds) return fail(T2_ERR_INVALID, "waveglow: row_seeds and an injected z exclude each other");
  if (a->z && wa->z_frames < frame0 + a->T_mel)
    return fail(T2_ERR_INVALID, "waveglow window: z holds %d frames, the window ends at frame %d", wa->z_frames,
                frame0 + a->T_mel);
  if (a->ws_bytes < waveglow_ws_bytes(m, a->B, a->T_mel)) return fail(T2_ERR_WORKSPACE, "waveglow workspace too small");
  const int B = a->B, T = a->T_mel, fp16 = m->fp16, passes = fp16 ? 1 : 3;
  const Dims d = dims_of(sh, B, T);
  Carve c(a->ws, 1024);
  WsLayout o;
  ws_layout(c, sh, B, T, &o);
  // Guard rows must read as zero: they are cleared here and only ever rewritten with zeros.  With per-flow ranges
  // (below) the rows a flow does not need are not rewritten and may hold stale values from earlier flows or calls
  // (skip and aud are not cleared at all); that is safe because no needed row reads an unneeded one.
  T2_CUDA(cudaMemsetAsync(o.spect, 0, planes_bytes(kCond, o.rows), s));
  T2_CUDA(cudaMemsetAsync(o.h, 0, planes_bytes(sh.C, o.rows), s));
  T2_CUDA(cudaMemsetAsync(o.acts, 0, planes_bytes(sh.C, o.rows), s));
  WG_STOP_POINT();
  // frame-domain planes: kFGuard zero rows before each sequence's frames and after them
  T2_TRY(tc_mel_to_planes(a->mel, a->io_half, B, T, a->lengths, kFGuard, d.spanf, o.x, o.x_rows, passes, s));
  // upsample + trim + unfold (glow.py:252-258)
  Main u;
  memset(&u, 0, sizeof(u));
  for (int j = 0; j < 4; ++j) u.seg[j] = Seg{o.x, o.x_rows, -j, 2};
  u.nseg = 4; u.nchunks = 8; u.row0 = kFGuard; u.wimg = m->up_img; u.n_tiles_m = d.ntf;
  u.B = B; u.span = d.spanf; u.T = T; u.lo = 0; u.hi = T;
  const UpsampleEpi::Params ue{m->up_bias, o.spect, o.rows, guard, d.span};
  WG_STOP_POINT();
  T2_TRY(gemm<UpsampleEpi>(u, ue, 80, fp16, s));

  // Per-flow column ranges.  The audio columns [32 out0, 32 out1) need the output of the flow that runs with n flows
  // still to follow over those columns widened by n * reach; that flow's WN layers run over one reach more.
  // Everything is clipped to the window: at a sequence edge the zero padding is the sequence's own.
  auto widen = [&](int n, int* lo, int* hi) {
    *lo = (int)std::max(0L, 32L * out0 - (long)reach * n);
    *hi = (int)std::min((long)d.L, 32L * out1 + (long)reach * n);
  };
  switch (sh.C) {
    case 128: T2_TRY(run_flows<128>(m, wa, o, d, widen, s)); break;
    case 256: T2_TRY(run_flows<256>(m, wa, o, d, widen, s)); break;
    case 384: T2_TRY(run_flows<384>(m, wa, o, d, widen, s)); break;
    default: T2_TRY(run_flows<512>(m, wa, o, d, widen, s)); break;
  }
  return T2_OK;
}

#ifdef T2_SELFTEST
int waveglow_state(T2WaveGlow* m, const T2WaveGlowWindowArgs* wa, int n_launches, float* spect, float* hbuf, float* acts,
                   float* skip, float* aud, cudaStream_t s) {
  if (!m) return fail(T2_ERR_INVALID, "waveglow: null argument");
  const Shape& sh = m->sh;
  if (n_launches < 0 || n_launches > launches_of(sh))
    return fail(T2_ERR_INVALID, "waveglow state: n_launches %d is not in [0, %d]", n_launches, launches_of(sh));
  g_launched = 0; g_stop_before = n_launches;
  const int r = waveglow_infer_window(m, wa, s);
  g_stop_before = -1;
  T2_TRY(r);
  const int B = wa->wg.B, T = wa->wg.T_mel, passes = m->fp16 ? 1 : 3;
  Carve c(wa->wg.ws, 1024);
  WsLayout o;
  ws_layout(c, sh, B, T, &o);
  const long n = (long)dims_of(sh, B, T).ntm * kTile;
  const unsigned blocks = (unsigned)((n + 127) / 128);
  const int guard = sh.guard();
  if (spect) unpack_planes_kernel<<<dim3(blocks, kCond / 8), 128, 0, s>>>(o.spect, o.rows, guard, passes, n, spect);
  if (hbuf) unpack_planes_kernel<<<dim3(blocks, sh.C / 8), 128, 0, s>>>(o.h, o.rows, guard, passes, n, hbuf);
  if (acts) unpack_planes_kernel<<<dim3(blocks, sh.C / 8), 128, 0, s>>>(o.acts, o.rows, guard, passes, n, acts);
  T2_CUDA(cudaGetLastError());
  if (skip) T2_CUDA(cudaMemcpyAsync(skip, o.skip, (size_t)n * sh.C * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (aud) T2_CUDA(cudaMemcpyAsync(aud, o.aud, (size_t)n * 8 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return T2_OK;
}
#endif

}  // namespace t2
