// The implicit GEMM on wgmma shared by the Tacotron2 convolutions (conv_tc.cu), WaveGlow (waveglow.cu) and the denoiser
// (denoiser.cu).
//
// A and the output are "k8 planes" (see conv_tc.cu): for each group of 8 channels a hi and a lo plane of [rows][8]
// fp16.  The GEMM's K is a list of segments, each a run of 64-channel chunks of some planes read at a row shift, so a
// strided or dilated convolution is one GEMM over shifted views of the same planes.  Every output row is computed
// from its own A rows in a fixed order, so a row gets the same bits wherever it sits in a tile.  The epilogue is
// chosen at compile time (EPI_*).
//
// The Tacotron2 convs (EPI_CONV) load one A tile of 132 rows per chunk instead: a k5 conv's 5 taps are that same tile
// addressed with the descriptor start shifted by tap * 16 bytes, so the tile crosses shared memory once per chunk.
//
// The HiFi-GAN convolutions (EPI_HIFI, hifigan.cu) have up to 15 taps: their K is seg[0]'s chunks read at ntaps row
// shifts seg[0].shift + tap * dil, tap-major.
//
// Tiers: fp32-grade = hi*hi + lo*hi + hi*lo (3 MMAs per K step); fp16 = hi*hi only, lo planes neither read nor written.
#pragma once
#include <float.h>
#include <string.h>

#include "common.cuh"
#include "umma.cuh"

namespace t2 {
namespace {

constexpr int kTile = 128;                  // output rows (group columns / frames / padded rows) per CTA
constexpr int kNT = 128, kWS = 4;           // MMA N per weight stage unless a caller picks another; weight ring stages
constexpr int kThreads = 384;               // warp 0 producer; warpgroups 1 / 2: MMA + epilogue
constexpr int kCluster = 2;                 // the CTAs of a cluster share each weight stage by multicast
constexpr unsigned long long kWd = 1ull << 32;
// Denoiser spectrum planes (EPI_SPECTRAL / EPI_PROJECT write them, EPI_OVERLAP's GEMM reads them): the real parts of the 513 bins
// in groups 0 ... 64, the imaginary parts in groups 65 ... 129, zero up to 136 groups = 17 whole 64-channel chunks.
constexpr int kBins = 513, kImGroup0 = 65, kSpecGroups = 136;
// Operand ranges (a split fp16 value overflows at 65504).  The audio is packed as it is, so its samples must stay below
// 65504 in magnitude.  The spectrum is stored as X / 512: |X| <= (sum of the window = 512) max |audio|, and the gate
// never raises it for strength >= 0, so the stored value is bounded by max |audio| as well.  The inverse basis
// (|w| <= 4.9e-4) is packed times 2^12 so that its lo halves stay out of fp16's subnormal range.  All three scales are
// powers of two; EPI_OVERLAP undoes them exactly.
constexpr float kSpecScale = 1.f / 512.f, kInvBasisScale = 4096.f;

__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t parity) {
  if (ptx::mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = clock64();
  while (!ptx::mbar_try_wait(bar, parity))
    if (clock64() - t0 > kWd) __trap();
}

enum { EPI_UPSAMPLE = 0, EPI_GATE = 1, EPI_RESSKIP = 2, EPI_SPECTRAL = 3, EPI_OVERLAP = 4, EPI_CONV = 5, EPI_PROJECT = 6,
       EPI_MAGPHASE = 7, EPI_HIFI = 8 };

// A tile rows beyond the output tile: EPI_CONV's tile m0 reads padded rows [m0 - 2, m0 + 130), every other epilogue
// 128 rows per segment.
constexpr int a_halo(int epi) { return epi == EPI_CONV ? 4 : 0; }
constexpr int a_stage_bytes(int epi) { return 16 * (kTile + a_halo(epi)) * 16; }   // 8 k8 groups x (hi, lo) of a chunk
constexpr int w_stage_bytes(int nt) { return nt * 64 * 2 * 2; }                    // hi + lo planes of nt rows x 64 k

struct Seg { const __half* planes; long rows; int shift, nchunks; };
struct GemmParams {
  Seg seg[4]; int nseg, nchunks;
  long row0;                        // plane row of tile row 0 of the A operands
  const uint8_t* wimg;
  int n_tiles_m, mt0;               // M tiles; the grid starts at tile mt0 (set by launch_gemm)
  int B, span, T; const int32_t* len; int len_mul;   // tile row q = b * span + t is data when t < T (and < len_b * len_mul)
  int lo, hi;                       // only rows with t in [lo, hi) are needed: a cluster holding none of them exits
  const float* bias;
  __half* out; long out_rows, out_row0;              // planes the epilogue writes
  float* skip; int first, res_cols;                  // RESSKIP: output columns < res_cols are the residual half
  int col_span;                                      // UPSAMPLE: span of the column domain
  float strength;                                    // SPECTRAL: the magnitude loses bias * strength
  float* audio; long audio_pitch;                    // OVERLAP: fp32 rows (B, audio_pitch); row t writes block t - lo
  const double* wsq;                                 // OVERLAP: the squared window (1024)
  const float* row_scale;                            // PROJECT: the target times row_scale[b]; MAGPHASE and (when set)
                                                     // OVERLAP: the output times row_scale[b].  Powers of two.
  const float* target;                               // PROJECT: magnitudes (B, 513, T - 1) fp32
  float* mag_out; float* phase_out;                  // MAGPHASE: (B, 513, T - 1) fp32
  // CONV: tile row q is padded row b * span + 2 + t (span = T + 4); y = act(acc * scale + bias), act 0 none, 1 relu,
  // 2 tanh; out_mode 0 writes the planes `out`, 1 fp32 rows (row of (b, t) = b * out_seq_rows + t, pitch ldo),
  // 2 fp32 (B, cout, T) plus the residual (B, T, cout); len: frames t >= len[b] are zeros in modes 0 and 2.
  int taps;                                          // CONV: 5 (conv k5) or 1 (a GEMM on the centre rows)
  const float* scale; int act, out_mode, cout;
  float* out_f32; long ldo; int out_seq_rows;
  const float* residual; long res_batch_stride;
  int skip_cols;                                     // RESSKIP: skip columns (the WN width); later columns are padding
  // HIFI: K = ntaps x seg[0]'s chunks, tap k at row shift seg[0].shift + k * dil.  Tile row q = b * span + t is input
  // row t; column n = phase * cout + channel is output row t * phases + phase, plane row out_row0 + b * col_span + that
  // (output rows >= col_span are not written).  Rows past len[b] * len_mul (or T * phases) are zeros.  x = acc + bias
  // (+ res_in) goes to x_out (or null); act planes `out` get lrelu(x, slope).  mrf (fp32, rows (b * col_span + row) x
  // cout): mrf = x (mrf_first) or mrf + x; with mrf_div > 0, `out` gets lrelu(mrf / mrf_div, slope) instead.
  int ntaps, dil, phases;
  const __half* res_in; __half* x_out;
  float* mrf; int mrf_first; float mrf_div, slope;
};

template <int PASSES>
__device__ __forceinline__ void store8(__half* planes, long rows, int grp, long row, const float* v) {
  __align__(16) __half hh[8];
  __align__(16) __half ll[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) split_fp16(v[i], hh[i], ll[i]);
  __half* dst = planes + (((long)grp * 2) * rows + row) * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hh);
  if (PASSES == 3) *reinterpret_cast<uint4*>(dst + rows * 8) = *reinterpret_cast<const uint4*>(ll);
}
template <int PASSES>
__device__ __forceinline__ void load8(const __half* planes, long rows, int grp, long row, float* v) {
  const __half* src = planes + (((long)grp * 2) * rows + row) * 8;
  __align__(16) __half hh[8];
  __align__(16) __half ll[8];
  *reinterpret_cast<uint4*>(hh) = *reinterpret_cast<const uint4*>(src);
  if (PASSES == 3) *reinterpret_cast<uint4*>(ll) = *reinterpret_cast<const uint4*>(src + rows * 8);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = __half2float(hh[i]) + (PASSES == 3 ? __half2float(ll[i]) : 0.f);
}

// does M tile mt hold a row q = b * span + t with b < B and t in [lo, hi)?
// (B * span <= 2^30, so int arithmetic suffices)
__device__ __forceinline__ bool tile_needed(const GemmParams& p, int mt) {
  if (mt >= p.n_tiles_m) return false;
  const int q0 = mt * kTile;
  for (int b = q0 / p.span; b < p.B && b * p.span < q0 + kTile; ++b) {
    const int s0 = b * p.span;
    if (max(q0 - s0, p.lo) < min(q0 + kTile - s0, p.hi)) return true;
  }
  return false;
}

// NT = MMA N per weight stage, NH = weight stages (N halves) per CTA column tile
template <int EPI, int PASSES, int NT = kNT, int NH = 2>
__global__ void __launch_bounds__(kThreads, 1) wg_gemm_kernel(const GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int kHalo = a_halo(EPI), kSeg = (kTile + kHalo) * 16, kAStage = a_stage_bytes(EPI);
  constexpr int kWStage = w_stage_bytes(NT), kOutPitch = NT * NH + 4;
  constexpr uint32_t kABytes = PASSES == 3 ? kAStage : kAStage / 2;
  constexpr uint32_t kWBytes = PASSES == 3 ? kWStage : kWStage / 2;   // the hi plane comes first in a stage
  // tap k reads the A tile from row tap0 + k; a single tap reads the centre rows of a halo tile
  const int taps = EPI == EPI_CONV ? p.taps : 1, tap0 = taps == 1 ? kHalo / 2 : 0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mt = p.mt0 + blockIdx.x, nt = blockIdx.y;
  // EPI_CONV computes every tile: its planes epilogue is what writes the zero padding rows the next layer reads
  if (EPI != EPI_CONV && (p.lo > 0 || p.hi < p.T)) {
    // both CTAs of a cluster take the same decision before any barrier: skip when neither tile holds a needed row.
    // A skipped tile writes nothing; its guard rows keep the zeros they were cleared to.  (With the full range every
    // launched cluster holds data rows.)
    const int c0 = p.mt0 + (int)(blockIdx.x & ~(unsigned)(kCluster - 1));
    bool need = false;
#pragma unroll
    for (int i = 0; i < kCluster; ++i) need = need || tile_needed(p, c0 + i);
    if (!need) return;
  }
  uint8_t* s_w = smem;
  uint8_t* s_a = smem + kWS * kWStage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_a + 2 * kAStage);
  uint64_t* a_full = bars; uint64_t* a_empty = bars + 2;
  uint64_t* w_full = bars + 4; uint64_t* w_empty = bars + 4 + kWS;
  const uint32_t rank = ptx::cluster_ctarank();
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) { ptx::mbar_init(&a_full[i], 1); ptx::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < kWS; ++i) { ptx::mbar_init(&w_full[i], 1); ptx::mbar_init(&w_empty[i], 2 * kCluster); }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::cluster_sync_all();
  const bool tile_live = mt < p.n_tiles_m;     // grid.x is rounded up to the cluster size

  if (warp == 0) {
    if (lane == 0) {
      const uint64_t pol_w = ptx::policy_evict_last(), pol_a = ptx::policy_evict_first();
      uint32_t wst = 0, wph = 0;
      const int mrow = tile_live ? mt : 0;     // dead tiles (cluster padding) stream tile 0 and discard
      for (int c = 0; c < p.nchunks; ++c) {
        const int sa = c & 1;
        wait_bar(&a_empty[sa], ((c >> 1) & 1) ^ 1);
        ptx::mbar_arrive_expect_tx(&a_full[sa], kABytes);
        const __half* base = nullptr; long rows = 0; int shift = 0, cc = 0, rem = c;
        bool found = false;
        if (EPI == EPI_HIFI) {
          const int tap = c / p.seg[0].nchunks;
          base = p.seg[0].planes; rows = p.seg[0].rows; shift = p.seg[0].shift + tap * p.dil; cc = c - tap * p.seg[0].nchunks;
        } else {
#pragma unroll
        for (int s = 0; s < 4; ++s)
          if (!found && s < p.nseg) {
            if (rem < p.seg[s].nchunks) { base = p.seg[s].planes; rows = p.seg[s].rows; shift = p.seg[s].shift; cc = rem; found = true; }
            else rem -= p.seg[s].nchunks;
          }
        }
        const long r0 = p.row0 + (long)mrow * kTile + shift;
        for (int g = 0; g < 8; ++g)
          for (int hl = 0; hl < (PASSES == 3 ? 2 : 1); ++hl) {
            const __half* src = base + (((long)(cc * 8 + g) * 2 + hl) * rows + r0) * 8;
            ptx::bulk_g2s_hint(s_a + sa * kAStage + (hl * 8 + g) * kSeg, src, kSeg, &a_full[sa], pol_a);
          }
        for (int th = 0; th < taps * NH; ++th) {
          const int tap = th / NH, h = th - tap * NH;
          wait_bar(&w_empty[wst], wph ^ 1);
          ptx::mbar_arrive_expect_tx(&w_full[wst], kWBytes);
          const uint8_t* wsrc = p.wimg + (((size_t)(nt * NH + h) * p.nchunks + c) * taps + tap) * kWStage;
          const uint32_t slice = kWBytes / kCluster;
          ptx::bulk_g2s_mc_hint(s_w + wst * kWStage + rank * slice, wsrc + rank * slice, slice, &w_full[wst],
                                (uint16_t)((1u << kCluster) - 1u), pol_w);
          if (++wst == kWS) { wst = 0; wph ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (tid >= 128) {
    const int wg = (tid >> 7) - 1, wt = tid & 127;
    float d[NH][NT / 2];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) d[h][i] = 0.f;
      ptx::wg_fence_regs<NT / 2>(d[h]);
    }
    uint32_t wst = 0, wph = 0;
    for (int c = 0; c < p.nchunks; ++c) {
      const int sa = c & 1;
      wait_bar(&a_full[sa], (c >> 1) & 1);
      const uint32_t ab = ptx::smem_u32(s_a + sa * kAStage) + (uint32_t)wg * (64 * 16);
      for (int tap = 0; tap < taps; ++tap) {
#pragma unroll
        for (int h = 0; h < NH; ++h) {
          wait_bar(&w_full[wst], wph);
          const uint32_t wb = ptx::smem_u32(s_w + wst * kWStage);
          ptx::wg_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t aoff = (2 * kk) * kSeg + (tap + tap0) * 16;
            const uint64_t a_hi = ptx::make_smem_desc(ab + aoff, kSeg, 128);
            const uint64_t b_hi = ptx::make_sw128_desc(wb + kk * 32);
            ptx::wgmma_f16<NT>(d[h], a_hi, b_hi);
            if (PASSES == 3) {
              const uint64_t a_lo = ptx::make_smem_desc(ab + 8 * kSeg + aoff, kSeg, 128);
              const uint64_t b_lo = ptx::make_sw128_desc(wb + NT * 128 + kk * 32);
              ptx::wgmma_f16<NT>(d[h], a_lo, b_hi);
              ptx::wgmma_f16<NT>(d[h], a_hi, b_lo);
            }
          }
          ptx::wg_commit();
          ptx::wg_wait<0>();
          ptx::wg_fence_regs<NT / 2>(d[h]);
          if (wt == 0)                       // this warpgroup is done with the weight stage in every CTA of the cluster
            for (int r = 0; r < kCluster; ++r) ptx::mbar_arrive_cluster(&w_empty[wst], r);
          if (++wst == kWS) { wst = 0; wph ^= 1; }
        }
      }
      if (wt == 0) ptx::mbar_arrive(&a_empty[sa]);
    }
    // every stage this CTA receives has been consumed: the operand stages become the fp32 output tile
    ptx::named_bar_sync(1, 256);
    float* s_out = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int i = 0; i < NT / 2; i += 2) {
        const int r = wg * 64 + ptx::wg_frag_row(i, wt), col = h * NT + ptx::wg_frag_col(i, wt);
        *reinterpret_cast<float2*>(s_out + r * kOutPitch + col) = make_float2(d[h][i], d[h][i + 1]);
      }
    ptx::named_bar_sync(1, 256);
    // ---- epilogue: thread = (tile row r, half of the columns) ----
    const int ct = tid - 128, r = ct & 127, half = ct >> 7;
    const long q = (long)mt * kTile + r;
    const int b = (int)(q / p.span), t = (int)(q - (long)b * p.span);
    const bool data = tile_live && b < p.B && t < p.T;
    const bool valid = data && (p.len == nullptr || t < p.len[b] * p.len_mul);
    const float* row = s_out + r * kOutPitch;
    if (tile_live) {
      if (EPI == EPI_GATE) {
        // columns [0, 128) of the tile are the tanh inputs of channels nt*128 + c, [128, 256) their sigmoid inputs
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
      } else if (EPI == EPI_RESSKIP) {
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
      } else if (EPI == EPI_UPSAMPLE) {    // tile column tile nt = mel channel, column = phase
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
      } else if (EPI == EPI_SPECTRAL || EPI == EPI_PROJECT) {
        // Denoiser forward transform, and Griffin-Lim's projection.  Columns [0, 128) of the tile are the real parts of
        // the bins nt * 128 + c, [128, 256) their imaginary parts.  Row t is frame t - 1 (t = 0: the zero frame before
        // the sequence).  SPECTRAL: mag' = max(|X| - strength * bias, 0); PROJECT: mag' = target[b, bin, t - 1] *
        // row_scale[b].  X' = X mag' / |X|, and (mag', 0) where |X| = 0 (atan2(0, 0) = 0).
        const bool live = valid && t >= 1;
        const float* tgt = EPI == EPI_PROJECT && live ? p.target + (long)b * kBins * (p.T - 1) + (t - 1) : nullptr;
        const float rs = EPI == EPI_PROJECT && live ? p.row_scale[b] : 0.f;
        for (int g = 0; g < 8; ++g) {
          const int j = nt * 16 + half * 8 + g;        // bins 8 j ... 8 j + 7
          float re[8], im[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float x = row[half * 64 + g * 8 + i], y = row[128 + half * 64 + g * 8 + i];
            const int bin = 8 * j + i;
            const float mag = sqrtf(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
            float m;
            if (EPI == EPI_PROJECT) {
              m = live && bin < kBins ? tgt[(long)bin * (p.T - 1)] * rs : 0.f;
            } else {
              const float bias = bin < kBins ? p.bias[bin] : 0.f;
              m = fmaxf(__fsub_rn(mag, __fmul_rn(bias, p.strength)), 0.f);
            }
            const float s = mag > 0.f ? m / mag : 0.f;
            re[i] = live ? (mag > 0.f ? x * s : m) * kSpecScale : 0.f;
            im[i] = live ? y * s * kSpecScale : 0.f;
          }
          if (j < kImGroup0) store8<PASSES>(p.out, p.out_rows, j, p.out_row0 + q, re);
          if (kImGroup0 + j < kSpecGroups) store8<PASSES>(p.out, p.out_rows, kImGroup0 + j, p.out_row0 + q, im);
        }
      } else if (EPI == EPI_MAGPHASE) {
        // Public STFT transform: columns as above; row t in [1, T) is frame t - 1 of the (B, 513, T - 1) outputs.  The
        // magnitude leaves the packing scale (row_scale[b] undoes it exactly); the phase does not depend on it.
        if (data && t >= 1) {
          const long F = p.T - 1;
          const float us = valid ? p.row_scale[b] : 0.f;
          float* mo = p.mag_out + (long)b * kBins * F + (t - 1);
          float* po = p.phase_out + (long)b * kBins * F + (t - 1);
          for (int c = 0; c < 64; ++c) {
            const int bin = nt * 128 + half * 64 + c;
            if (bin >= kBins) break;
            const float x = row[half * 64 + c], y = row[128 + half * 64 + c];
            mo[(long)bin * F] = valid ? sqrtf(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))) * us : 0.f;
            po[(long)bin * F] = valid ? atan2f(y, x) : 0.f;
          }
        }
      } else if (EPI == EPI_OVERLAP) {
        // Denoiser / STFT inverse transform.  Row t is block t of the trimmed output: the MMA has already added the four
        // frames t - 1 ... t + 2 that overlap it.  p.len[b] = 1 + the number of frames of row b (frame f exists when
        // f >= 0 and f + 1 < len); its output ends at block len - 2.
        if (b < p.B && t >= p.lo && t < p.hi) {
          const int fend = p.len[b];
          const bool in_row = t + 2 < fend;
          float* dst = p.audio + (long)b * p.audio_pitch + 256L * (t - p.lo) + half * 128;
          for (int c = 0; c < 128; c += 4) {
            float v[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int col = half * 128 + c + i;
              // window_sumsquare: a float32 sum, one frame at a time in frame order, each add done in double
              float env = 0.f;
#pragma unroll
              for (int f = t - 1; f <= t + 2; ++f)
                if (f >= 0 && f + 1 < fend) env = (float)((double)env + p.wsq[256 * (t + 2 - f) + col]);
              float y = row[col] * (1.f / (kSpecScale * kInvBasisScale));
              if (p.row_scale) y *= p.row_scale[b];
              if (env > FLT_MIN) y = y / env;
              v[i] = in_row ? y * 4.f : 0.f;
            }
            *reinterpret_cast<float4*>(dst + c) = make_float4(v[0], v[1], v[2], v[3]);
          }
        }
      } else if (EPI == EPI_HIFI) {
        // thread = (tile row r, half of the columns)
        constexpr int kHalf = NT * NH / 2;
        if (b < p.B) {
          const long lout = (long)p.T * p.phases;
          const long lim = p.len ? min(lout, (long)max(p.len[b], 0) * p.len_mul) : lout;
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
      } else if (EPI == EPI_CONV) {
        // thread = (tile row r, every other group of 8 columns); frame pt of sequence b is tile row q
        const int pt = t - 2;
        const bool in_seq = b < p.B && pt >= 0 && pt < p.T;
        // planes output: frames t >= len[b] are written as zeros, the padding a sequence of that length has alone
        const bool in_len = in_seq && (p.out_mode != 0 || p.len == nullptr || pt < p.len[b]);
        const int n0 = nt * NT * NH;
        for (int c0 = half * 8; c0 < NT * NH; c0 += 16) {
          float v[8];
          const float4 v0 = *reinterpret_cast<const float4*>(row + c0);
          const float4 v1 = *reinterpret_cast<const float4*>(row + c0 + 4);
          v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
          if (n0 + c0 >= p.cout) continue;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int n = n0 + c0 + i;
            float x = v[i] * p.scale[n] + p.bias[n];
            if (p.act == 1) x = fmaxf(x, 0.f);
            else if (p.act == 2) x = tanhf(x);
            v[i] = in_len ? x : 0.f;
          }
          if (p.out_mode == 0) {          // next layer's planes (zeros in the padding rows); plane row = q + 2
            const int g = (n0 + c0) >> 3;
            store8<3>(p.out, p.out_rows, g, q + 2, v);
            // the 2 guard rows at both ends of the plane stay zero
            if (q == 0 || q == (long)p.n_tiles_m * kTile - 1) {
              const float z[8] = {};
              const long gr = q == 0 ? 0 : q + 3;
              for (int k = 0; k < 2; ++k) store8<3>(p.out, p.out_rows, g, gr + k, z);
            }
          } else if (in_seq && p.out_mode == 1) {   // fp32 rows (b * out_seq_rows + t, ldo)
            float* o = p.out_f32 + ((long)b * p.out_seq_rows + pt) * p.ldo + n0 + c0;
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
          } else if (in_seq && p.out_mode == 2) {   // (B, cout, T) + residual (B, T, cout), masked beyond len
            const bool keep = p.len == nullptr || pt < p.len[b];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int n = n0 + c0 + i;
              float x = v[i];
              if (p.residual) x += p.residual[(long)b * p.res_batch_stride + (long)pt * p.cout + n];
              p.out_f32[((long)b * p.cout + n) * p.T + pt] = keep ? x : 0.f;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  // peers' consumers arrive on our w_empty barriers: drain before leaving (producer thread state is gone here, so wait
  // on the parity each barrier reaches after its last use)
  if (tid == 0) {
    const int total = p.nchunks * taps * NH;
    for (int i = 0; i < kWS; ++i) {
      const int uses = (total - i + kWS - 1) / kWS;
      if (uses > 0) wait_bar(&w_empty[i], (uses - 1) & 1);
    }
  }
  __syncthreads();
  ptx::cluster_sync_all();
}

template <int EPI, int PASSES, int NT = kNT, int NH = 2>
int launch_gemm(GemmParams p, int n_tiles_n, cudaStream_t s) {
  constexpr int kOperands = kWS * w_stage_bytes(NT) + 2 * a_stage_bytes(EPI);
  static_assert(kTile * (NT * NH + 4) * 4 <= kOperands, "output tile reuses the operand stages");
  const size_t smem = (size_t)kOperands + (4 + 2 * kWS) * 8 + 64;
  T2_CUDA(cudaFuncSetAttribute(wg_gemm_kernel<EPI, PASSES, NT, NH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  // the grid spans the tiles from the first needed row (sequence 0, t = lo) to the last (sequence B-1, t = hi-1)
  p.mt0 = p.lo / kTile;
  const int last = (int)(((long)(p.B - 1) * p.span + p.hi - 1) / kTile);
  const int gx = ((last - p.mt0 + 1 + kCluster - 1) / kCluster) * kCluster;
  cfg.gridDim = dim3(gx, n_tiles_n); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeClusterDimension;
  at.val.clusterDim.x = kCluster; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
  cfg.attrs = &at; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, wg_gemm_kernel<EPI, PASSES, NT, NH>, p);
  if (e != cudaSuccess) return fail(T2_ERR_CUDA, "wgmma gemm launch failed: %s", cudaGetErrorString(e));
  g_launch_count++;
  return T2_OK;
}

template <int EPI>
int gemm(const GemmParams& p, int n_tiles_n, bool fp16, cudaStream_t s) {
  return fp16 ? launch_gemm<EPI, 1>(p, n_tiles_n, s) : launch_gemm<EPI, 3>(p, n_tiles_n, s);
}

}  // namespace
}  // namespace t2
