// HiFi-GAN generator inference (jik876/hifi-gan, models.py: Generator, ResBlock1, ResBlock2) on sm_90a.
//
// Every convolution except conv_post is one implicit GEMM on wgmma (wg_gemm_kernel, HiFiEpi) over k8 planes (see
// wg_gemm.cuh): for each group of 8 channels a hi and a lo plane of [rows][8] fp16, one row per sample at the stage's
// rate.  A k-tap dilated Conv1d is K = k taps x ceil(C_in / 64) chunks of the same planes read at the row shifts
// tap * d - pad.  A ConvTranspose1d of stride u, kernel 2u and padding u / 2 is polyphase: output sample q u + r reads
// input frames q - 1, q and q + 1 (two of them with a non-zero weight), so it is one GEMM over those three shifts whose
// N stacks the u phases, column n = r * C_out + channel, and whose epilogue scatters row q to rows q u + r.
//
// Rows: sequence b's sample t of stage s is row guard + b * span_s + t, span_s = rate_s T_mel + guard.  The guard rows
// after every sequence (and before the first) are zero: the zero padding of the widest convolution.  With lengths,
// the rows t >= rate_s lengths[b] are written as zeros too, so a row sees exactly the padding it has alone, and every
// output row sums its products in one order wherever it sits in a tile.
//
// Fusions (the epilogue of every GEMM):
//   conv_pre           lrelu(x, 0.1) planes: ups[0]'s input.
//   ups[i]             x (the resblocks' common residual) and lrelu(x, 0.1) planes.
//   resblock convs     x = conv + residual, written as x (the next residual) and lrelu(x, 0.1) (the next input); the
//                      last conv of resblock j adds x into one fp32 MRF sum in j order instead, and the last
//                      resblock's writes lrelu(sum / n_kernels) with slope 0.1 (the next ups' input) or 0.01 (conv_post's).
//   conv_post          (N = 1) a CUDA-core kernel: tanh, fp32 or fp16 audio (B, 256 T_mel).
//
// Buffers: five plane slots (x of ups, lrelu of ups, the running residual, two activations) sized for the largest
// stage and re-laid out at every stage; each GEMM writes every row of its outputs from the first sequence's row to the
// last sequence's guard.  When an input slot takes a new layout, the rows before the first sequence and the channels
// that pad C to whole 64-channel chunks are cleared.
//
// Tiers: fp32-grade = split-fp16 planes and weights (3 MMAs per K step); fp16 = hi planes and weights only.  The MRF
// sum and conv_post are fp32 in both.
#include <string.h>

#include <algorithm>
#include <vector>

#include "conv_tc.h"
#include "wg_gemm.cuh"

namespace t2 {
namespace {

constexpr int kPreK = 7, kPostK = 7, kMelGroups = 16;   // conv_pre / conv_post kernels; 80 mels padded to 128 channels
constexpr int kSlots = 5;
enum { kY = 0, kAY = 1, kX = 2, kA = 3, kT = 4 };     // slots: ups x, lrelu(ups x), residual, activations A and T

// A supported configuration (hifigan_shape): every size below follows from it.
struct Net {
  int rb, n_up, up[T2_HIFIGAN_MAX_STAGES], C0, nk, rk[T2_HIFIGAN_MAX_KERNELS], rd[T2_HIFIGAN_MAX_KERNELS][3];
  int guard;                                                   // zero rows around each sequence: the widest padding
  int ch(int s) const { return s < 0 ? C0 : C0 >> (s + 1); }  // channels at stage s (-1: conv_pre's output)
  int rate(int s) const { int r = 1; for (int i = 0; i <= s; ++i) r *= up[i]; return r; }
  int nd() const { return rb == 1 ? 3 : 2; }                   // dilations per resblock
  int convs_per_rb() const { return rb == 1 ? 6 : 2; }
  int n_convs() const { return 2 + n_up + n_up * nk * convs_per_rb(); }   // conv_pre, ups, resblock convs, conv_post
  int num_weights() const { return 3 * n_convs(); }
  int rb_conv(int i, int j, int which) const { return 1 + n_up + (i * nk + j) * convs_per_rb() + which; }
};

// one convolution as the engine runs it
struct Conv {
  int cin, cout, k, dil, pad;      // Conv1d: the taps read rows tap * dil - pad; ConvTranspose1d: 3 shifts from -1
  int up;                          // 0: Conv1d; u: ConvTranspose1d of stride u
  int ntaps, cin_pad, ncols, n_pad, nt_rows;   // GEMM: K = ntaps x cin_pad, N = ncols padded to n_pad
  uint8_t* img; float* bias;
  long K() const { return (long)ntaps * cin_pad; }
};

Conv make_conv(int cin, int cout, int k, int dil, int up) {
  Conv c;
  memset(&c, 0, sizeof(c));
  c.cin = cin; c.cout = cout; c.k = k; c.dil = dil; c.up = up;
  c.pad = up ? 1 : (k * dil - dil) / 2;
  c.ntaps = up ? 3 : k;
  c.cin_pad = (cin + 63) / 64 * 64;
  c.ncols = (up ? up : 1) * cout;
  c.nt_rows = c.ncols <= 64 ? 64 : 128;           // N per weight stage; a CTA takes 1 stage (<= 128) or 2 columns
  const int cta_cols = c.ncols <= 128 ? c.nt_rows : 256;
  c.n_pad = (c.ncols + cta_cols - 1) / cta_cols * cta_cols;
  return c;
}

}  // namespace
}  // namespace t2

struct T2HiFiGAN {
  int fp16;
  t2::Net net;
  std::vector<t2::Conv> convs;    // table order: conv_pre, ups, resblock convs (conv_post is the post_* fields)
  float* post_w = nullptr;        // conv_post: weight (C, 7), folded, then the bias
  float* tmp = nullptr;           // fp32 staging of the matrix being packed
  float* scale = nullptr;         // the weight-norm scale of each dim-0 row
};

namespace t2 {
namespace {

const char* hifigan_shape(const T2HiFiGANConfig* c, Net* n) {
  memset(n, 0, sizeof(*n));
  if (c->n_mel_channels != kMel) return "n_mel_channels must be 80";
  if (c->resblock != 1 && c->resblock != 2) return "resblock must be \"1\" or \"2\"";
  if (c->n_upsamples < 1 || c->n_upsamples > T2_HIFIGAN_MAX_STAGES) return "upsample_rates must have 1 ... 8 entries";
  long prod = 1;
  for (int i = 0; i < c->n_upsamples; ++i) {
    const int u = c->upsample_rates[i];
    if (u < 2 || u % 2) return "upsample_rates must be even";
    if (c->upsample_kernel_sizes[i] != 2 * u) return "upsample_kernel_sizes must be twice upsample_rates";
    prod *= u;
    if (prod > 256) break;
  }
  if (prod != 256) return "the product of upsample_rates must be 256 (the hop length)";
  const int C0 = c->upsample_initial_channel;
  if (C0 < 8 || C0 > 512 || C0 % 8) return "upsample_initial_channel must be a multiple of 8 in 8 ... 512";
  for (int i = 0; i < c->n_upsamples; ++i) {
    const int ci = C0 >> (i + 1);
    if (ci < 8 || ci % 8 || (ci << (i + 1)) != C0)
      return "every stage's channels (upsample_initial_channel / 2^(i+1)) must be a multiple of 8 in 8 ... 512";
  }
  if (c->n_kernels < 1 || c->n_kernels > T2_HIFIGAN_MAX_KERNELS) return "resblock_kernel_sizes must have 1 ... 8 entries";
  n->rb = c->resblock; n->n_up = c->n_upsamples; n->C0 = C0; n->nk = c->n_kernels;
  int guard = std::max(kPreK / 2, kPostK / 2) + 1;
  for (int j = 0; j < n->nk; ++j) {
    const int k = c->resblock_kernel_sizes[j];
    if (k < 1 || k > 15 || k % 2 == 0) return "resblock_kernel_sizes must be odd and at most 15";
    n->rk[j] = k;
    for (int m = 0; m < n->nd(); ++m) {
      const int d = c->resblock_dilation_sizes[j][m];
      if (d < 1 || (long)(k - 1) * d / 2 > T2_HIFIGAN_MAX_PAD)
        return "resblock_dilation_sizes must be >= 1 with (kernel - 1) * dilation / 2 <= 64";
      n->rd[j][m] = d;
      guard = std::max(guard, (k - 1) * d / 2);
    }
  }
  for (int i = 0; i < n->n_up; ++i) n->up[i] = c->upsample_rates[i];
  if (c->fp16 != 0 && c->fp16 != 1) return "fp16 must be 0 or 1";
  n->guard = guard;
  return nullptr;
}

std::vector<Conv> conv_list(const Net& n) {
  std::vector<Conv> v;
  v.push_back(make_conv(kMel, n.C0, kPreK, 1, 0));
  for (int i = 0; i < n.n_up; ++i) v.push_back(make_conv(n.ch(i - 1), n.ch(i), 2 * n.up[i], 1, n.up[i]));
  for (int i = 0; i < n.n_up; ++i)
    for (int j = 0; j < n.nk; ++j)
      for (int w = 0; w < n.convs_per_rb(); ++w) {
        const int m = w % n.nd(), d = w < n.nd() ? n.rd[j][m] : 1;   // ResBlock1: convs1 dilated, convs2 dilation 1
        v.push_back(make_conv(n.ch(i), n.ch(i), n.rk[j], d, 0));
      }
  return v;
}

// ---- per-stage sizes ------------------------------------------------------------------------------------
struct Stage {
  int R, C, L, span, ntm;   // rate (samples per mel frame), channels, samples per sequence, row span, M tiles
  long rows;                // plane rows: guard + ntm tiles + guard
  int cpad;                 // channels padded to whole 64-channel chunks
};
Stage stage(const Net& n, int s, int B, int T) {
  Stage g;
  g.R = s < 0 ? 1 : n.rate(s);
  g.C = n.ch(s);
  g.L = g.R * T;
  g.span = g.L + n.guard;
  g.ntm = (int)(((long)B * g.span + kTile - 1) / kTile);
  g.rows = 2L * n.guard + (long)g.ntm * kTile;
  g.cpad = (g.C + 63) / 64 * 64;
  return g;
}

struct WsLayout { __half* mel; long mel_rows; int mel_span; __half* slot[kSlots]; float* mrf; };
void ws_layout(Carve& c, const Net& n, int B, int T, WsLayout* o) {
  const Stage f = stage(n, -1, B, T);
  o->mel_rows = f.rows; o->mel_span = f.span;
  o->mel = c.take<__half>(planes_bytes(kMelGroups * 8, f.rows) / sizeof(__half), 1024);
  size_t slot = 0, mrf = 0;
  for (int s = -1; s < n.n_up; ++s) {
    const Stage g = stage(n, s, B, T);
    slot = std::max(slot, planes_bytes(g.cpad, g.rows));
    if (s >= 0) mrf = std::max(mrf, (size_t)g.ntm * kTile * g.C);
  }
  for (int i = 0; i < kSlots; ++i) o->slot[i] = c.take<__half>(slot / sizeof(__half), 1024);
  o->mrf = c.take<float>(mrf, 1024);
}

// ---- kernels ---------------------------------------------------------------------------------------------
// the weight-norm scale g / ||v|| of dim-0 row blockIdx.x of v (1 when g is null: the weight is plain); 128 threads
__global__ void wn_scale_kernel(const void* v, const void* g, int per_row, int half, float* scale) {
  __shared__ double red[4];
  const long n = blockIdx.x;
  if (g == nullptr) {
    if (threadIdx.x == 0) scale[n] = 1.f;
    return;
  }
  double ss = 0.0;
  for (int i = threadIdx.x; i < per_row; i += blockDim.x) { const double x = ldw(v, n * per_row + i, half); ss += x * x; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) scale[n] = (float)((double)ldw(g, n, half) / sqrt(red[0] + red[1] + red[2] + red[3]));
}

// GEMM weight row n (of n_pad), K index tap * cin_pad + ci.  Conv1d: v (cout, cin, k) times the scale of row n.
// ConvTranspose1d: column n = r * cout + co; tap s reads input frame q + s - 1, which output q u + r reaches through
// kernel index j = (1 - s) u + r + u / 2 (zero outside [0, 2u)); v (cin, cout, 2u) times the scale of row ci.
__global__ void build_conv_kernel(const void* v, const void* b, const float* scale, int cin, int cout, int k, int up,
                                  int cin_pad, int ncols, int half, float* w, float* bias) {
  const int n = blockIdx.x;
  const int ntaps = up ? 3 : k;
  const long K = (long)ntaps * cin_pad;
  for (long kk = threadIdx.x; kk < K; kk += blockDim.x) {
    const int tap = (int)(kk / cin_pad), ci = (int)(kk - (long)tap * cin_pad);
    float x = 0.f;
    if (n < ncols && ci < cin) {
      if (!up) {
        x = ldw(v, ((long)n * cin + ci) * k + tap, half) * scale[n];
      } else {
        const int r = n / cout, co = n - r * cout, j = (1 - tap) * up + r + up / 2;
        if (j >= 0 && j < 2 * up) x = ldw(v, ((long)ci * cout + co) * 2 * up + j, half) * scale[ci];
      }
    }
    w[(long)n * K + kk] = x;
  }
  if (n == 0)
    for (int c = threadIdx.x; c < cout; c += blockDim.x) bias[c] = ldw(b, c, half);
}

// conv_post: w (C, 7) times the scale of its one output row, then the bias
__global__ void build_post_kernel(const void* v, const void* b, const float* scale, int C, int half, float* w) {
  for (int i = threadIdx.x; i < C * kPostK; i += blockDim.x) w[i] = ldw(v, i, half) * scale[0];
  if (threadIdx.x == 0) w[C * kPostK] = ldw(b, 0, half);
}

__device__ __forceinline__ long clamp_len(const int32_t* len, int b, int T) {
  return len == nullptr ? T : (long)min(max(len[b], 0), T);
}

// ---- the GEMM epilogue ----------------------------------------------------------------------------------
// Tile row q = b * span + t is input row t; column n = phase * cout + channel is output row t * phases + phase, plane
// row out_row0 + b * col_span + that (output rows >= col_span are not written).  Rows past len[b] * len_mul (or
// T * phases) are zeros.  x = acc + bias (+ res_in) goes to x_out (or null); act planes `out` get lrelu(x, slope).
// mrf (fp32, rows (b * col_span + row) x cout): mrf = x (mrf_first) or mrf + x; with mrf_div > 0, `out` gets
// lrelu(mrf / mrf_div, slope) instead.
struct HiFiEpi : EpiDefaults {
  static constexpr KForm kK = KForm::kTapShifts;
  struct Params {
    const float* bias; __half* out; long out_rows, out_row0; int col_span;
    int phases, cout;
    const __half* res_in; __half* x_out;
    float* mrf; int mrf_first; float mrf_div, slope;
  };
  template <int PASSES, int NT, int NH>
  static __device__ __forceinline__ void apply(const Main& m, const Params& p, const float* row, int r, int half, long q,
                                               int b, int t, int nt, bool data, bool valid) {
    // thread = (tile row r, half of the columns)
    constexpr int kHalf = NT * NH / 2;
    if (b < m.B) {
      const long lout = (long)m.T * p.phases;
      const long lim = m.len ? min(lout, (long)max(m.len[b], 0) * m.len_mul) : lout;
      for (int g = 0; g < kHalf / 8; ++g) {
        const int cl = half * kHalf + g * 8, n = nt * NT * NH + cl;
        if (n >= p.phases * p.cout) break;
        const int ph = n / p.cout, ch = n - ph * p.cout;
        const long to = (long)t * p.phases + ph;
        if (to >= p.col_span) continue;
        const bool live = to < lim;
        const long orow = p.out_row0 + (long)b * p.col_span + to;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = row[cl + i] + p.bias[ch + i];
        if (p.res_in) {
          float rv[8];
          load8<PASSES>(p.res_in, p.out_rows, ch >> 3, orow, rv);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] += rv[i];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = live ? v[i] : 0.f;
        if (p.x_out) store8<PASSES>(p.x_out, p.out_rows, ch >> 3, orow, v);
        if (p.mrf) {
          float4* sm = reinterpret_cast<float4*>(p.mrf + ((long)b * p.col_span + to) * p.cout + ch);
          float4 s0 = make_float4(v[0], v[1], v[2], v[3]), s1 = make_float4(v[4], v[5], v[6], v[7]);
          if (!p.mrf_first) {
            const float4 o0 = sm[0], o1 = sm[1];
            s0 = make_float4(o0.x + v[0], o0.y + v[1], o0.z + v[2], o0.w + v[3]);
            s1 = make_float4(o1.x + v[4], o1.y + v[5], o1.z + v[6], o1.w + v[7]);
          }
          if (p.mrf_div > 0.f) {
            v[0] = s0.x / p.mrf_div; v[1] = s0.y / p.mrf_div; v[2] = s0.z / p.mrf_div; v[3] = s0.w / p.mrf_div;
            v[4] = s1.x / p.mrf_div; v[5] = s1.y / p.mrf_div; v[6] = s1.z / p.mrf_div; v[7] = s1.w / p.mrf_div;
          } else {
            sm[0] = s0; sm[1] = s1;
          }
        }
        if (p.out) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = v[i] > 0.f ? v[i] : v[i] * p.slope;
          store8<PASSES>(p.out, p.out_rows, ch >> 3, orow, v);
        }
      }
    }
  }
};

// conv_post + tanh (models.py Generator.forward's last lines) on CUDA cores: one thread per output sample, its
// C x 7 products summed in channel-major, tap-minor order; samples >= 256 lengths[b] are zero
template <int PASSES>
__global__ void __launch_bounds__(256) conv_post_kernel(const __half* __restrict__ planes, long rows, int guard, int span,
                                                        int B, int L, int T, const int32_t* __restrict__ len,
                                                        const float* __restrict__ w, int C, void* audio, int io_half) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * L) return;
  const int b = (int)(i / L), t = (int)(i - (long)b * L);
  const long row = guard + (long)b * span + t;
  float acc = 0.f;
  for (int g = 0; g < C / 8; ++g) {
    float v[kPostK][8];
#pragma unroll
    for (int k = 0; k < kPostK; ++k) load8<PASSES>(planes, rows, g, row + k - kPostK / 2, v[k]);
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int k = 0; k < kPostK; ++k) acc = fmaf(__ldg(&w[(g * 8 + c) * kPostK + k]), v[k][c], acc);
  }
  const float y = t < clamp_len(len, b, T) * (L / T) ? tanhf(acc + __ldg(&w[C * kPostK])) : 0.f;
  if (io_half) reinterpret_cast<__half*>(audio)[i] = __float2half_rn(y);
  else reinterpret_cast<float*>(audio)[i] = y;
}

int check_weights(const Net& n, const void* const* w, int count) {
  if (count != n.num_weights())
    return fail(T2_ERR_INVALID, "hifigan: expected %d weight pointers, got %d", n.num_weights(), count);
  for (int i = 0; i < count; ++i)
    if (w[i] == nullptr && i % 3 != 1) return fail(T2_ERR_INVALID, "hifigan: weight %d is null", i);
  return T2_OK;
}

int pack(T2HiFiGAN* m, const void* const* w, cudaStream_t s) {
  const int half = m->fp16;
  for (size_t i = 0; i < m->convs.size(); ++i) {
    const Conv& c = m->convs[i];
    const void* const* e = w + 3 * i;     // bias, weight_g, weight_v
    const int rows0 = c.up ? c.cin : c.cout, per_row = c.up ? c.cout * c.k : c.cin * c.k;
    wn_scale_kernel<<<rows0, 128, 0, s>>>(e[2], e[1], per_row, half, m->scale);
    T2_LAUNCH_CHECK();
    build_conv_kernel<<<c.n_pad, 256, 0, s>>>(e[2], e[0], m->scale, c.cin, c.cout, c.k, c.up, c.cin_pad, c.ncols, half,
                                               m->tmp, c.bias);
    T2_LAUNCH_CHECK();
    T2_TRY(tc_pack_weights(m->tmp, c.n_pad, (int)c.K(), 1, c.nt_rows, c.img, s));
  }
  const void* const* e = w + 3 * m->convs.size();
  const int C = m->net.ch(m->net.n_up - 1);
  wn_scale_kernel<<<1, 128, 0, s>>>(e[2], e[1], C * kPostK, half, m->scale);
  T2_LAUNCH_CHECK();
  build_post_kernel<<<1, 256, 0, s>>>(e[2], e[0], m->scale, C, half, m->post_w);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int destroy(T2HiFiGAN* m) {
  if (!m) return T2_OK;
  for (Conv& c : m->convs) { cudaFree(c.img); cudaFree(c.bias); }
  cudaFree(m->post_w); cudaFree(m->tmp); cudaFree(m->scale);
  delete m;
  return T2_OK;
}

size_t ws_bytes(const T2HiFiGAN* m, int B, int T) {
  Carve c(nullptr, 1024);
  WsLayout o;
  ws_layout(c, m->net, B, T, &o);
  return c.bytes();
}

template <int PASSES>
int gemm_hifi(const Main& g, const HiFiEpi::Params& e, const Conv& c, cudaStream_t s) {
  if (c.nt_rows == 64) return launch_gemm<HiFiEpi, PASSES, 64, 1>(g, e, c.n_pad / 64, s);
  if (c.ncols <= 128) return launch_gemm<HiFiEpi, PASSES, 128, 1>(g, e, c.n_pad / 128, s);
  return launch_gemm<HiFiEpi, PASSES, 128, 2>(g, e, c.n_pad / 256, s);
}

// the GEMM of convolution c from planes `in` (stage layout si) to stage layout so's outputs
struct Io {
  const __half* in; const __half* res; __half* x; __half* act; float* mrf;
  int mrf_first; float mrf_div, slope;
};
int run_conv(const T2HiFiGAN* m, const Conv& c, const Stage& si, const Stage& so, int B, const int32_t* len, const Io& io,
             cudaStream_t s) {
  Main g;
  memset(&g, 0, sizeof(g));
  const int G = m->net.guard;
  g.seg[0] = Seg{io.in, si.rows, c.up ? -1 : -c.pad, c.cin_pad / 64};
  g.nseg = 1; g.dil = c.up ? 1 : c.dil; g.nchunks = c.ntaps * (c.cin_pad / 64);
  g.row0 = G; g.wimg = c.img; g.n_tiles_m = si.ntm;
  // every row up to the last sequence's guard is written, so that the guard rows are zero in this layout too
  g.B = B; g.span = si.span; g.T = si.L; g.lo = 0; g.hi = si.span;
  g.len = len; g.len_mul = so.R;
  const HiFiEpi::Params e{c.bias, io.act, so.rows, G, so.span, c.up ? c.up : 1, c.cout, io.res, io.x,
                          io.mrf, io.mrf_first, io.mrf_div, io.slope};
  return m->fp16 ? gemm_hifi<1>(g, e, c, s) : gemm_hifi<3>(g, e, c, s);
}

// What a GEMM reads of a slot in stage layout st that no epilogue writes: rows [0, guard), before the first sequence,
// and every row of the padding channels [C, cpad) (zero weights, but stale bits could be NaN or Inf)
int clear_unwritten(__half* planes, const Stage& st, int guard, cudaStream_t s) {
  const size_t group_bytes = (size_t)2 * st.rows * 16;
  T2_CUDA(cudaMemset2DAsync(planes, (size_t)st.rows * 16, 0, (size_t)guard * 16, (size_t)(st.C / 8) * 2, s));
  if (st.C < st.cpad)
    T2_CUDA(cudaMemsetAsync((char*)planes + (st.C / 8) * group_bytes, 0, (size_t)(st.cpad - st.C) / 8 * group_bytes, s));
  return T2_OK;
}

int infer(T2HiFiGAN* m, const T2HiFiGANArgs* a, cudaStream_t s) {
  if (!m || !a || !a->mel || !a->audio || !a->ws) return fail(T2_ERR_INVALID, "hifigan: null argument");
  const Net& n = m->net;
  const int B = a->B, T = a->T_mel, G = n.guard;
  if (B <= 0 || T <= 0) return fail(T2_ERR_INVALID, "hifigan: empty input (B=%d, T_mel=%d)", B, T);
  if (a->io_half != 0 && a->io_half != 1) return fail(T2_ERR_INVALID, "hifigan: io_half must be 0 or 1");
  if ((long)B * (256L * T + G) >= (1L << 30))
    return fail(T2_ERR_INVALID, "hifigan: B * (256 T_mel + %d) must stay below 2^30 (B=%d, T_mel=%d)", G, B, T);
  if (a->ws_bytes < ws_bytes(m, B, T)) return fail(T2_ERR_WORKSPACE, "hifigan workspace too small");
  const int passes = m->fp16 ? 1 : 3;
  Carve c(a->ws, 1024);
  WsLayout o;
  ws_layout(c, n, B, T, &o);
  __half* const* sl = o.slot;
  T2_TRY(tc_mel_to_planes(a->mel, a->io_half, B, T, a->lengths, G, o.mel_span, o.mel, o.mel_rows, passes, s));
  const Stage f = stage(n, -1, B, T);
  Stage mel_st = f;
  mel_st.rows = o.mel_rows; mel_st.cpad = kMelGroups * 8;
  // conv_pre -> lrelu(x, 0.1) into A
  T2_TRY(clear_unwritten(sl[kA], f, G, s));
  Io io;
  memset(&io, 0, sizeof(io));
  io.in = o.mel; io.act = sl[kA]; io.slope = 0.1f;
  T2_TRY(run_conv(m, m->convs[0], mel_st, f, B, a->lengths, io, s));
  int act = kA;           // the slot holding the current stage input's lrelu planes
  Stage prev = f;
  for (int i = 0; i < n.n_up; ++i) {
    const Stage st = stage(n, i, B, T);
    // ups[i]: x into Y, lrelu(x, 0.1) into AY
    memset(&io, 0, sizeof(io));
    io.in = sl[act]; io.x = sl[kY]; io.act = sl[kAY]; io.slope = 0.1f;
    T2_TRY(clear_unwritten(sl[kAY], st, G, s));
    T2_TRY(run_conv(m, m->convs[1 + i], prev, st, B, a->lengths, io, s));
    T2_TRY(clear_unwritten(sl[kA], st, G, s));
    T2_TRY(clear_unwritten(sl[kT], st, G, s));
    const bool last_stage = i == n.n_up - 1;
    for (int j = 0; j < n.nk; ++j) {
      int in = kAY;       // resblock j reads lrelu(ups x); its residual starts at ups x
      const int n_conv = n.convs_per_rb();
      for (int w = 0; w < n_conv; ++w) {
        // ResBlock1 runs convs1[m], convs2[m] for m = 0, 1, 2; ResBlock2 convs[m] for m = 0, 1
        const int mm = n.rb == 1 ? w / 2 : w;
        const bool second = n.rb == 1 ? w % 2 == 1 : true;    // adds the residual
        const int idx = n.rb_conv(i, j, n.rb == 1 ? (second ? 3 + mm : mm) : mm);
        const int out = in == kA ? kT : kA;
        memset(&io, 0, sizeof(io));
        io.in = sl[in]; io.slope = 0.1f;
        if (second) io.res = sl[mm == 0 ? kY : kX];
        if (w == n_conv - 1) {
          io.mrf = o.mrf; io.mrf_first = j == 0;
          if (j == n.nk - 1) { io.mrf_div = (float)n.nk; io.act = sl[out]; io.slope = last_stage ? 0.01f : 0.1f; }
        } else {
          io.act = sl[out];
          if (second) io.x = sl[kX];
        }
        T2_TRY(run_conv(m, m->convs[idx], st, st, B, a->lengths, io, s));
        in = out;
      }
      if (j == n.nk - 1) act = in;
    }
    prev = st;
  }
  const long total = (long)B * prev.L;
  const int C = prev.C;
  if (m->fp16)
    conv_post_kernel<1><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(sl[act], prev.rows, G, prev.span, B, prev.L, T,
                                                                       a->lengths, m->post_w, C, a->audio, a->io_half);
  else
    conv_post_kernel<3><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(sl[act], prev.rows, G, prev.span, B, prev.L, T,
                                                                       a->lengths, m->post_w, C, a->audio, a->io_half);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace
}  // namespace t2

using namespace t2;

extern "C" {

int32_t t2_hifigan_num_weights(const T2HiFiGANConfig* cfg) {
  Net n;
  return cfg && hifigan_shape(cfg, &n) == nullptr ? n.num_weights() : 0;
}

int t2_hifigan_create(T2HiFiGAN** out, const T2HiFiGANConfig* cfg, const void* const* weights, int32_t n_weights,
                      void* stream) {
  if (!out || !cfg || !weights) return fail(T2_ERR_INVALID, "hifigan: null argument");
  Net n;
  if (const char* why = hifigan_shape(cfg, &n))
    return fail(T2_ERR_UNSUPPORTED, "hifigan: the sm_90a kernels do not support this configuration: %s", why);
  T2_TRY(check_weights(n, weights, n_weights));
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0)
    return fail(T2_ERR_UNSUPPORTED, "libt2b200 is built for sm_90a only (device is sm_%d%d)", p.major, p.minor);
  T2HiFiGAN* m = new T2HiFiGAN();
  m->fp16 = cfg->fp16;
  m->net = n;
  m->convs = conv_list(n);
  size_t tmp = 0;
  bool ok = true;
  for (Conv& c : m->convs) {
    tmp = std::max(tmp, (size_t)c.n_pad * c.K());
    ok = ok && cudaMalloc((void**)&c.img, tc_weights_bytes(c.n_pad, (int)c.K(), 1, c.nt_rows)) == cudaSuccess &&
         cudaMalloc((void**)&c.bias, c.cout * sizeof(float)) == cudaSuccess;
  }
  const int C = n.ch(n.n_up - 1);
  ok = ok && cudaMalloc((void**)&m->tmp, tmp * sizeof(float)) == cudaSuccess &&
       cudaMalloc((void**)&m->scale, 1024 * sizeof(float)) == cudaSuccess &&
       cudaMalloc((void**)&m->post_w, (C * kPostK + 1) * sizeof(float)) == cudaSuccess;
  int r = ok ? pack(m, weights, (cudaStream_t)stream)
             : fail(T2_ERR_CUDA, "hifigan: out of device memory for the packed weights");
  if (r != T2_OK) { destroy(m); return r; }
  *out = m;
  return T2_OK;
}

int t2_hifigan_refresh(T2HiFiGAN* h, const void* const* weights, int32_t n_weights, void* stream) {
  if (!h || !weights) return fail(T2_ERR_INVALID, "hifigan: null argument");
  T2_TRY(check_weights(h->net, weights, n_weights));
  return pack(h, weights, (cudaStream_t)stream);
}

int t2_hifigan_destroy(T2HiFiGAN* h) { return destroy(h); }

size_t t2_hifigan_workspace_bytes(const T2HiFiGAN* h, int32_t B, int32_t T_mel) {
  return h && B > 0 && T_mel > 0 ? ws_bytes(h, B, T_mel) : 0;
}

int t2_hifigan_infer(T2HiFiGAN* h, const T2HiFiGANArgs* a, void* stream) { return infer(h, a, (cudaStream_t)stream); }

}  // extern "C"
