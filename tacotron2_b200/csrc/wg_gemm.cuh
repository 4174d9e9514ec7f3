// The implicit GEMM on wgmma shared by the Tacotron2 convolutions (conv_tc.cu), WaveGlow (waveglow.cu), the denoiser,
// STFT and Griffin-Lim (denoiser.cu) and HiFi-GAN (hifigan.cu).  This header holds the main loop; each caller defines
// the epilogues of its GEMMs next to the code that reads their outputs.
//
// A and the output are "k8 planes" (see conv_tc.cu): for each group of 8 channels a hi and a lo plane of [rows][8]
// fp16.  Every output row is computed from its own A rows in a fixed order, so a row gets the same bits wherever it
// sits in a tile.  The GEMM's K takes one of three forms, which the epilogue type selects (Epi::kK):
//   KForm::kSegments   a list of segments, each a run of 64-channel chunks of some planes read at a row shift, so a
//                      strided or dilated convolution is one GEMM over shifted views of the same planes;
//   KForm::kHaloTile   one A tile of 132 rows per chunk (seg[0]); the m.taps weight stages of a chunk (a k5 conv's 5
//                      taps) address that same tile with the descriptor start shifted by tap * 16 bytes, so the tile
//                      crosses shared memory once per chunk;
//   KForm::kTapShifts  seg[0]'s chunks read at row shifts seg[0].shift + tap * m.dil, tap-major (up to 15 taps).
//
// An epilogue type Epi provides
//   struct Params                      what its epilogue reads;
//   static constexpr KForm kK          the K form (EpiDefaults: kSegments);
//   static constexpr bool kSkipTiles   whether clusters holding no row with t in [m.lo, m.hi) exit at once
//                                      (EpiDefaults: true);
//   template <int PASSES, int NT, int NH> static __device__ __forceinline__ void apply(const Main& m,
//       const Params& e, const float* row, int r, int half, long q, int b, int t, int nt, bool data, bool valid)
//                                      called once per thread of the MMA warpgroups with its tile row (r, of
//                                      NT * NH fp32 columns in shared memory) and half of the columns.
//
// Tiers: fp32-grade = hi*hi + lo*hi + hi*lo (3 MMAs per K step); fp16 = hi*hi only, lo planes neither read nor written.
#pragma once
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

__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t parity) {
  if (ptx::mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = clock64();
  while (!ptx::mbar_try_wait(bar, parity))
    if (clock64() - t0 > kWd) __trap();
}

enum class KForm { kSegments, kHaloTile, kTapShifts };
struct EpiDefaults {
  static constexpr KForm kK = KForm::kSegments;
  static constexpr bool kSkipTiles = true;
};

// A tile rows beyond the output tile: a halo tile m0 reads padded rows [m0 - 2, m0 + 130), the other forms 128 rows
// per segment.
constexpr int a_halo(KForm k) { return k == KForm::kHaloTile ? 4 : 0; }
constexpr int a_stage_bytes(KForm k) { return 16 * (kTile + a_halo(k)) * 16; }   // 8 k8 groups x (hi, lo) of a chunk
constexpr int w_stage_bytes(int nt) { return nt * 64 * 2 * 2; }                  // hi + lo planes of nt rows x 64 k

struct Seg { const __half* planes; long rows; int shift, nchunks; };
// What the main loop reads: the producer, the MMA warpgroups and each epilogue thread's row and validity.
struct Main {
  Seg seg[4]; int nseg, nchunks;
  long row0;                        // plane row of tile row 0 of the A operands
  const uint8_t* wimg;
  int n_tiles_m, mt0;               // M tiles; the grid starts at tile mt0 (set by launch_gemm)
  int B, span, T; const int32_t* len; int len_mul;   // tile row q = b * span + t is data when t < T (and < len_b * len_mul)
  int lo, hi;                       // only rows with t in [lo, hi) are needed: a cluster holding none of them exits
  int taps;                         // kHaloTile: weight stages (taps) per chunk, 5 (conv k5) or 1 (the centre rows)
  int dil;                          // kTapShifts: the row step between taps
};

// The kernel's one argument.  (As two kernel arguments, Main and Params compiled to different code: the epilogues
// read their fields through a pointer into the parameter space, with more instructions and, for the 80-column conv,
// 4 more registers.)
template <class Epi>
struct GemmArgs { Main m; typename Epi::Params e; };

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
__device__ __forceinline__ bool tile_needed(const Main& p, int mt) {
  if (mt >= p.n_tiles_m) return false;
  const int q0 = mt * kTile;
  for (int b = q0 / p.span; b < p.B && b * p.span < q0 + kTile; ++b) {
    const int s0 = b * p.span;
    if (max(q0 - s0, p.lo) < min(q0 + kTile - s0, p.hi)) return true;
  }
  return false;
}

// NT = MMA N per weight stage, NH = weight stages (N halves) per CTA column tile
template <class Epi, int PASSES, int NT = kNT, int NH = 2>
__global__ void __launch_bounds__(kThreads, 1) wg_gemm_kernel(const GemmArgs<Epi> args) {
  const Main& p = args.m;
  const typename Epi::Params& e = args.e;
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int kHalo = a_halo(Epi::kK), kSeg = (kTile + kHalo) * 16, kAStage = a_stage_bytes(Epi::kK);
  constexpr int kWStage = w_stage_bytes(NT), kOutPitch = NT * NH + 4;
  constexpr uint32_t kABytes = PASSES == 3 ? kAStage : kAStage / 2;
  constexpr uint32_t kWBytes = PASSES == 3 ? kWStage : kWStage / 2;   // the hi plane comes first in a stage
  // tap k reads the A tile from row tap0 + k; a single tap reads the centre rows of a halo tile
  const int taps = Epi::kK == KForm::kHaloTile ? p.taps : 1, tap0 = taps == 1 ? kHalo / 2 : 0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mt = p.mt0 + blockIdx.x, nt = blockIdx.y;
  if (Epi::kSkipTiles && (p.lo > 0 || p.hi < p.T)) {
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
        if (Epi::kK == KForm::kTapShifts) {
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
    if (tile_live) Epi::template apply<PASSES, NT, NH>(p, e, s_out + r * kOutPitch, r, half, q, b, t, nt, data, valid);
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

template <class Epi, int PASSES, int NT = kNT, int NH = 2>
int launch_gemm(Main p, const typename Epi::Params& e, int n_tiles_n, cudaStream_t s) {
  constexpr int kOperands = kWS * w_stage_bytes(NT) + 2 * a_stage_bytes(Epi::kK);
  static_assert(kTile * (NT * NH + 4) * 4 <= kOperands, "output tile reuses the operand stages");
  const size_t smem = (size_t)kOperands + (4 + 2 * kWS) * 8 + 64;
  T2_CUDA(cudaFuncSetAttribute(wg_gemm_kernel<Epi, PASSES, NT, NH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
  const cudaError_t err = cudaLaunchKernelEx(&cfg, wg_gemm_kernel<Epi, PASSES, NT, NH>, GemmArgs<Epi>{p, e});
  if (err != cudaSuccess) return fail(T2_ERR_CUDA, "wgmma gemm launch failed: %s", cudaGetErrorString(err));
  g_launch_count++;
  return T2_OK;
}

template <class Epi>
int gemm(const Main& p, const typename Epi::Params& e, int n_tiles_n, bool fp16, cudaStream_t s) {
  return fp16 ? launch_gemm<Epi, 1>(p, e, n_tiles_n, s) : launch_gemm<Epi, 3>(p, e, n_tiles_n, s);
}

}  // namespace
}  // namespace t2
