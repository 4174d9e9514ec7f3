// Tensor-core conv1d / GEMM for the Encoder (model.py:157-167, 174-175), the BiLSTM input projection
// (model.py:169-171) and the Postnet (model.py:112-146): split-fp16 implicit GEMM on wgmma.
//
//   out[(b,t), n] = epilogue( sum_{tap, ci} W[n][tap][ci] * x[(b, t + tap - pad), ci] )
//
// * Activations live in "k8 planes": for every group of 8 channels, a hi plane and a lo plane of
//   [rows][8] fp16 (16 bytes per row).  Rows are the sequences with 2 zero rows before and after each
//   (+2 guard rows at both ends of the plane), so a 128-row output tile needs input rows [m0-2, m0+130):
//   ONE contiguous 2112-byte bulk copy per plane, and the 5 taps of a conv are the SAME shared-memory
//   tile addressed with the descriptor start shifted by tap*16 bytes -- no im2col, 5x reuse from SMEM.
//   (K-major no-swizzle canonical layout with LBO = 2112 between k8 groups, SBO = 128 between 8-row groups.)
// * Weights are packed per (n-tile, 64-channel chunk, tap) as [hi | lo] SWIZZLE_128B planes and streamed
//   through a ring; within a cluster of 2 CTAs the weight stage is fetched once and TMA-multicast.
// * fp32-grade: hi*hi + lo*hi + hi*lo, 3 MMAs (M=64 per warpgroup, N=n_tile, K=16) per 16 channels, fp32 in registers.
// * Epilogue: folded BatchNorm scale/shift (+bias), ReLU / tanh, and either the next layer's planes,
//   fp32 rows (LSTM gate pre-activations) or the final (B, 80, T) tensor with the residual (model.py:511/524).
#include <stdlib.h>
#include <string.h>

#include "conv_tc.h"
#include "umma.cuh"

namespace t2 {
namespace {

constexpr int kTile = 128;                 // output rows per CTA
constexpr int kHalo = 4;                   // input rows = kTile + 4
constexpr int kSeg = (kTile + kHalo) * 16; // bytes of one k8 plane segment of a tile = 2112
constexpr int kAStage = 16 * kSeg;         // 8 k8 groups x (hi, lo) = 33792 bytes per 64-channel chunk
constexpr int kThreadsC = 384;             // warp 0 producer; warpgroups 1 / 2: MMA + epilogue
constexpr int kCluster = 2;                // CTAs of a cluster share each weight stage by multicast
constexpr unsigned long long kWd = 1ull << 32;

__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t parity) {
  if (ptx::mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = clock64();
  while (!ptx::mbar_try_wait(bar, parity))
    if (clock64() - t0 > kWd) __trap();
}

struct ConvParams {
  const __half* in; long in_plane_rows;      // rows_alloc of the input planes
  const uint8_t* wimg;
  int nchunks, taps;                          // chunks of 64 input channels; 5 or 1
  int B, T, seq_pad;                          // seq_pad = 4: padded row p = b*(T+4) + 2 + t
  int n_tiles_m;
  const float* scale; const float* shift;     // per output channel
  int act, out_mode, cout;
  __half* out_planes; long out_plane_rows;
  float* out_f32; long ldo; int out_seq_rows;  // out_mode 1: row of (b, t) = b * out_seq_rows + t
  const float* residual; long res_batch_stride; const int32_t* row_len;
};

template <int NT, int NH, int WS>   // NT = weight rows per stage (MMA N), NH = n-halves per CTA, WS = weight stages
__global__ void __launch_bounds__(kThreadsC, 1) conv_tc_kernel(const ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int kWStage = NT * 64 * 2 * 2;   // hi + lo planes of NT rows x 64 k
  constexpr int kOutPitch = NT * NH + 4;     // fp32 output tile [128][kOutPitch] (reuses the operand stages)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mt = blockIdx.x, nt = blockIdx.y;
  uint8_t* s_w = smem;                                   // WS x kWStage (1024-aligned: SWIZZLE_128B)
  uint8_t* s_a = smem + WS * kWStage;                    // 2 x kAStage
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_a + 2 * kAStage);
  uint64_t* a_full = bars; uint64_t* a_empty = bars + 2;
  uint64_t* w_full = bars + 4; uint64_t* w_empty = bars + 4 + WS;
  const uint32_t rank = ptx::cluster_ctarank();
  if (tid == 0) {
    // a stage is released by the 2 MMA warpgroups (a weight stage: of every CTA of the cluster)
    for (int i = 0; i < 2; ++i) { ptx::mbar_init(&a_full[i], 1); ptx::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < WS; ++i) { ptx::mbar_init(&w_full[i], 1); ptx::mbar_init(&w_empty[i], 2 * kCluster); }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::cluster_sync_all();
  const bool tile_live = mt < p.n_tiles_m;     // grid.x is rounded up to the cluster size

  if (warp == 0) {
    if (lane == 0) {
      const uint64_t pol_w = ptx::policy_evict_last(), pol_a = ptx::policy_evict_first();
      uint32_t wst = 0, wph = 0;
      for (int c = 0; c < p.nchunks; ++c) {
        const int sa = c & 1;
        wait_bar(&a_empty[sa], ((c >> 1) & 1) ^ 1);
        ptx::mbar_arrive_expect_tx(&a_full[sa], kAStage);
        const int mrow = tile_live ? mt : 0;   // dead tiles (cluster padding) stream tile 0 and discard
        for (int g = 0; g < 8; ++g)
          for (int hl = 0; hl < 2; ++hl) {
            const __half* src = p.in + (((long)(c * 8 + g) * 2 + hl) * p.in_plane_rows + (long)mrow * kTile) * 8;
            ptx::bulk_g2s_hint(s_a + sa * kAStage + (hl * 8 + g) * kSeg, src, kSeg, &a_full[sa], pol_a);
          }
        for (int th = 0; th < p.taps * NH; ++th) {
          const int tap = th / NH, h = th - tap * NH;
          wait_bar(&w_empty[wst], wph ^ 1);
          ptx::mbar_arrive_expect_tx(&w_full[wst], kWStage);
          const uint8_t* wsrc = p.wimg + (((size_t)(nt * NH + h) * p.nchunks + c) * p.taps + tap) * kWStage;
          const uint32_t slice = kWStage / kCluster;
          ptx::bulk_g2s_mc_hint(s_w + wst * kWStage + rank * slice, wsrc + rank * slice, slice, &w_full[wst],
                                (uint16_t)((1u << kCluster) - 1u), pol_w);
          if (++wst == WS) { wst = 0; wph ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (tid >= 128) {
    // ---- MMA warpgroups 1 / 2: output rows [64 wg, 64 wg + 64) of the tile, all NT * NH columns in registers ----
    const int wg = (tid >> 7) - 1, wt = tid & 127;
    float d[NH][NT / 2];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) d[h][i] = 0.f;
      ptx::wg_fence_regs<NT / 2>(d[h]);
    }
    uint32_t wst = 0, wph = 0;
    const int tap0 = p.taps == 1 ? 2 : 0;   // a GEMM (taps == 1) reads the centre rows of the halo tile
    for (int c = 0; c < p.nchunks; ++c) {
      const int sa = c & 1;
      wait_bar(&a_full[sa], (c >> 1) & 1);
      const uint32_t ab = ptx::smem_u32(s_a + sa * kAStage) + (uint32_t)wg * (64 * 16);
      for (int tap = 0; tap < p.taps; ++tap) {
#pragma unroll
        for (int h = 0; h < NH; ++h) {
          wait_bar(&w_full[wst], wph);
          const uint32_t wb = ptx::smem_u32(s_w + wst * kWStage);
          ptx::wg_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t aoff = (2 * kk) * kSeg + (tap + tap0) * 16;
            const uint64_t a_hi = ptx::make_smem_desc(ab + aoff, kSeg, 128);
            const uint64_t a_lo = ptx::make_smem_desc(ab + 8 * kSeg + aoff, kSeg, 128);
            const uint64_t b_hi = ptx::make_sw128_desc(wb + kk * 32);
            const uint64_t b_lo = ptx::make_sw128_desc(wb + NT * 128 + kk * 32);
            ptx::wgmma_f16<NT>(d[h], a_hi, b_hi);
            ptx::wgmma_f16<NT>(d[h], a_lo, b_hi);
            ptx::wgmma_f16<NT>(d[h], a_hi, b_lo);
          }
          ptx::wg_commit();
          ptx::wg_wait<0>();
          ptx::wg_fence_regs<NT / 2>(d[h]);
          if (wt == 0)                       // this warpgroup is done with the weight stage in every CTA of the cluster
            for (int r = 0; r < kCluster; ++r) ptx::mbar_arrive_cluster(&w_empty[wst], r);
          if (++wst == WS) { wst = 0; wph ^= 1; }
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
    // ---- epilogue: thread = (output row r of the tile, half of the 8-column groups) ----
    const int ct = tid - 128, r = ct & 127, chalf = ct >> 7;
    const long prow = (long)mt * kTile + r;          // padded row index p
    const int span = p.T + p.seq_pad;
    const int b = (int)(prow / span), pt = (int)(prow - (long)b * span) - p.seq_pad / 2;
    const bool valid = tile_live && b < p.B && pt >= 0 && pt < p.T;
    // planes output: frames t >= row_len[b] are written as zeros, the padding a sequence of that length has alone
    const bool in_len = valid && (p.out_mode != 0 || p.row_len == nullptr || pt < p.row_len[b]);
    const int n0 = nt * NT * NH;
    if (tile_live) {
      for (int c0 = chalf * 8; c0 < NT * NH; c0 += 16) {
        float v[8];
        const float4 v0 = *reinterpret_cast<const float4*>(s_out + r * kOutPitch + c0);
        const float4 v1 = *reinterpret_cast<const float4*>(s_out + r * kOutPitch + c0 + 4);
        v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
        if (n0 + c0 >= p.cout) continue;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int n = n0 + c0 + i;
          float x = v[i] * p.scale[n] + p.shift[n];
          if (p.act == 1) x = fmaxf(x, 0.f);
          else if (p.act == 2) x = tanhf(x);
          v[i] = in_len ? x : 0.f;
        }
        if (p.out_mode == 0) {          // next layer's planes (zeros in the padding rows)
          __align__(16) __half hh[8];
          __align__(16) __half ll[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) split_fp16(v[i], hh[i], ll[i]);
          const long g = (n0 + c0) >> 3;
          __half* dst = p.out_planes + ((g * 2) * p.out_plane_rows + prow + 2) * 8;
          *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hh);
          *reinterpret_cast<uint4*>(dst + p.out_plane_rows * 8) = *reinterpret_cast<const uint4*>(ll);
          // guard rows at both ends of the plane stay zero
          if (prow == 0 || prow == (long)p.n_tiles_m * kTile - 1) {
            const uint4 z = make_uint4(0, 0, 0, 0);
            const long gr = prow == 0 ? 0 : prow + 3;
            for (int q = 0; q < 2; ++q) {
              __half* gd = p.out_planes + ((g * 2) * p.out_plane_rows + gr + q) * 8;
              *reinterpret_cast<uint4*>(gd) = z;
              *reinterpret_cast<uint4*>(gd + p.out_plane_rows * 8) = z;
            }
          }
        } else if (valid && p.out_mode == 1) {   // fp32 rows (b*T + t, ldo)
          float* o = p.out_f32 + ((long)b * p.out_seq_rows + pt) * p.ldo + n0 + c0;
          *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
        } else if (valid && p.out_mode == 2) {   // (B, cout, T) + residual (B, T, cout), masked beyond row_len
          const bool keep = p.row_len == nullptr || pt < p.row_len[b];
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
  __syncthreads();
  // peers' consumers arrive on our w_empty barriers: drain before leaving (producer thread state is
  // gone here, so wait on the parity each barrier reaches after its last use)
  if (tid == 0) {
    const int total = p.nchunks * p.taps * NH;
    for (int i = 0; i < WS; ++i) {
      const int uses = (total - i + WS - 1) / WS;       // number of times stage i was filled
      if (uses > 0) wait_bar(&w_empty[i], (uses - 1) & 1);
    }
  }
  __syncthreads();
  ptx::cluster_sync_all();
}

// ---- layout conversion kernels ---------------------------------------------------------------------
// fp32 channels-last rows (B, T, C) [batch stride] -> k8 planes with sequence padding; frames t >= len
// and channels >= C are zero; every row of every plane (incl. guards) is written.
__global__ void rows_to_planes_kernel(const float* __restrict__ x, long batch_stride, int C, int c_pad,
                                      const int32_t* __restrict__ len, int B, int T, __half* __restrict__ planes,
                                      long plane_rows, const float* __restrict__ in_scale) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;     // plane row (incl. 2 guard rows)
  const int g = blockIdx.y;
  if (row >= plane_rows) return;
  const long prow = row - 2;
  const int span = T + 4;
  __align__(16) __half hh[8];
  __align__(16) __half ll[8];
  int b = -1, t = -1;
  if (prow >= 0) { b = (int)(prow / span); t = (int)(prow - (long)b * span) - 2; }
  const bool valid = b >= 0 && b < B && t >= 0 && t < T && (len == nullptr || t < len[b]);
  const float mul = in_scale ? *in_scale : 1.f;       // power-of-two pre-scale (gradients do not fit fp16 otherwise)
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    const float v = (valid && c < C) ? x[(long)b * batch_stride + (long)t * C + c] * mul : 0.f;
    split_fp16(v, hh[i], ll[i]);
  }
  __half* dst = planes + (((long)g * 2) * plane_rows + row) * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hh);
  *reinterpret_cast<uint4*>(dst + plane_rows * 8) = *reinterpret_cast<const uint4*>(ll);
}

// embedding gather straight into planes (model.py:503 / 518); symbols at t >= len[b] are not read, their rows are zero
__global__ void embed_to_planes_kernel(const int64_t* __restrict__ text, const float* __restrict__ emb, int n_symbols,
                                       const int32_t* __restrict__ len, int B, int T, __half* __restrict__ planes,
                                       long plane_rows) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y;
  if (row >= plane_rows) return;
  const long prow = row - 2;
  const int span = T + 4;
  int b = -1, t = -1;
  if (prow >= 0) { b = (int)(prow / span); t = (int)(prow - (long)b * span) - 2; }
  const bool valid = b >= 0 && b < B && t >= 0 && t < T && (len == nullptr || t < len[b]);
  __align__(16) __half hh[8];
  __align__(16) __half ll[8];
  long id = 0;
  if (valid) { id = text[(long)b * T + t]; id = id < 0 ? 0 : (id >= n_symbols ? n_symbols - 1 : id); }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float v = valid ? emb[id * kEnc + g * 8 + i] : 0.f;
    split_fp16(v, hh[i], ll[i]);
  }
  __half* dst = planes + (((long)g * 2) * plane_rows + row) * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hh);
  *reinterpret_cast<uint4*>(dst + plane_rows * 8) = *reinterpret_cast<const uint4*>(ll);
}

// W (cout, cin, taps) fp32 [or (cout, cin) when taps == 1] -> per (n-tile, chunk, tap) [hi | lo] SWIZZLE_128B
// planes of NT rows x 64 channels; rows >= cout and channels >= cin are zero.
__global__ void pack_conv_w_kernel(const float* __restrict__ w, int cout, int cin, int taps, int nt_rows,
                                   int nchunks, uint8_t* __restrict__ img) {
  const int tap = blockIdx.x % taps, c = (blockIdx.x / taps) % nchunks, nt = blockIdx.x / (taps * nchunks);
  __half* hi = reinterpret_cast<__half*>(img + (size_t)blockIdx.x * nt_rows * 256);
  __half* lo = hi + nt_rows * 64;
  for (int i = threadIdx.x; i < nt_rows * 64; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    const int n = nt * nt_rows + r, ci = c * 64 + k;
    const float v = (n < cout && ci < cin) ? w[((long)n * cin + ci) * taps + tap] : 0.f;
    __half h, l;
    split_fp16(v, h, l);
    const uint32_t e = img_elem_offset(r, k);
    hi[e] = h; lo[e] = l;
  }
}

__global__ void fold_bn_bias_kernel(const float* cbias, const float* g, const float* b, const float* mean,
                                    const float* var, float eps, float* scale, float* shift, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (g == nullptr) { scale[c] = 1.f; shift[c] = cbias ? cbias[c] : 0.f; return; }
  const float s = g[c] / sqrtf(var[c] + eps);
  scale[c] = s;
  shift[c] = b[c] + ((cbias ? cbias[c] : 0.f) - mean[c]) * s;
}

template <int NT, int NH, int WS>
int launch_conv(const ConvParams& p, int n_tiles_n, cudaStream_t s) {
  constexpr int kWStage = NT * 64 * 2 * 2;
  const size_t smem = (size_t)WS * kWStage + 2 * kAStage + (4 + 2 * WS) * 8 + 64;
  T2_CUDA(cudaFuncSetAttribute(conv_tc_kernel<NT, NH, WS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  const int gx = ((p.n_tiles_m + kCluster - 1) / kCluster) * kCluster;
  cfg.gridDim = dim3(gx, n_tiles_n); cfg.blockDim = dim3(kThreadsC); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeClusterDimension;
  at.val.clusterDim.x = kCluster; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
  cfg.attrs = &at; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, conv_tc_kernel<NT, NH, WS>, p);
  if (e != cudaSuccess) return fail(T2_ERR_CUDA, "conv_tc launch failed: %s", cudaGetErrorString(e));
  g_launch_count++;
  return T2_OK;
}

}  // namespace

// ---- host API -------------------------------------------------------------------------------------
long tc_plane_rows(int B, int T) {
  const long rpad = (long)B * (T + 4);
  return 4 + ((rpad + kTile - 1) / kTile) * kTile;
}
size_t tc_planes_bytes(int B, int T, int c_pad) { return (size_t)(c_pad / 8) * 2 * tc_plane_rows(B, T) * 16; }

int tc_pack_weights(const float* w, int cout, int cin, int taps, int nt_rows, uint8_t** img, cudaStream_t s) {
  const int nchunks = (cin + 63) / 64, n_tiles_n = (cout + nt_rows - 1) / nt_rows;
  const size_t bytes = (size_t)n_tiles_n * nchunks * taps * nt_rows * 256;
  if (!*img) T2_CUDA(cudaMalloc((void**)img, bytes));
  pack_conv_w_kernel<<<n_tiles_n * nchunks * taps, 256, 0, s>>>(w, cout, cin, taps, nt_rows, nchunks, *img);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_rows_to_planes_scaled(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                             __half* planes, const float* in_scale, cudaStream_t s) {
  const long rows = tc_plane_rows(B, T);
  rows_to_planes_kernel<<<dim3((unsigned)((rows + 127) / 128), c_pad / 8), 128, 0, s>>>(x, batch_stride, C, c_pad, len, B, T,
                                                                                      planes, rows, in_scale);
  T2_LAUNCH_CHECK();
  return T2_OK;
}
int tc_rows_to_planes(const float* x, long batch_stride, int C, int c_pad, const int32_t* len, int B, int T,
                      __half* planes, cudaStream_t s) {
  return tc_rows_to_planes_scaled(x, batch_stride, C, c_pad, len, B, T, planes, nullptr, s);
}

int tc_embed_to_planes(const int64_t* text, const float* emb, int n_symbols, const int32_t* len, int B, int T,
                       __half* planes, cudaStream_t s) {
  const long rows = tc_plane_rows(B, T);
  embed_to_planes_kernel<<<dim3((unsigned)((rows + 127) / 128), kEnc / 8), 128, 0, s>>>(text, emb, n_symbols, len, B, T,
                                                                                       planes, rows);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_fold_bn(const float* cbias, const float* g, const float* b, const float* mean, const float* var, float eps,
               float* scale, float* shift, int C, cudaStream_t s) {
  fold_bn_bias_kernel<<<(C + 127) / 128, 128, 0, s>>>(cbias, g, b, mean, var, eps, scale, shift, C);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int tc_conv(const TcConvArgs& a, cudaStream_t s) {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.in = a.in; p.in_plane_rows = tc_plane_rows(a.B, a.T);
  p.wimg = a.wimg; p.nchunks = a.cin_pad / 64; p.taps = a.taps;
  p.B = a.B; p.T = a.T; p.seq_pad = 4;
  p.n_tiles_m = (int)((p.in_plane_rows - 4) / kTile);
  p.scale = a.scale; p.shift = a.shift; p.act = a.act; p.out_mode = a.out_mode; p.cout = a.cout;
  p.out_planes = a.out_planes; p.out_plane_rows = p.in_plane_rows;
  p.out_f32 = a.out_f32; p.ldo = a.ldo; p.out_seq_rows = a.out_seq_rows > 0 ? a.out_seq_rows : a.T;
  p.residual = a.residual; p.row_len = a.row_len;
  p.res_batch_stride = a.res_batch_stride ? a.res_batch_stride : (long)a.T * a.cout;
  // weights are packed in stages of nt_rows rows; a CTA covers 2 stages' worth of columns when cout allows
  if (a.nt_rows == 128) return launch_conv<128, 2, 4>(p, (a.cout + 255) / 256, s);
  if (a.nt_rows == 80) return launch_conv<80, 1, 4>(p, (a.cout + 79) / 80, s);
  return fail(T2_ERR_INVALID, "tc_conv: unsupported n-tile %d", a.nt_rows);
}

}  // namespace t2
