// Time-batched weight gradients of the two decoder LSTMs on the tensor cores (wgmma, split fp16):
//     dW[g][k] = sum over all (t, b) of dG[t, b, g] * X[t, b, k]            (4096 x 1792 and 4096 x 2560, K = T x B)
// One decoder step = one K chunk of 64 batch rows.  Both operands are turned into K-major SWIZZLE_128B operand
// images once (rows = gates / input features, K = batch row of one step): dG^T scaled per gate row by a power of two
// (max over all steps in [0.5, 1): gradients span many orders of magnitude, fp16 does not), X^T as is.  A CTA owns a
// 128 (gates) x 256 (features) tile of one K split (kWgSeg steps), streams [A hi|lo 32 KB][B hi|lo 64 KB] stages and
// issues hi.hi + hi.lo + lo.hi per 16-wide K step into 128 x 256 fp32 register accumulators (two warpgroups of 64 gate
// rows each); the K splits are added by a
// reduce kernel in a fixed order (bit-reproducible, and the accumulation chains stay short).
// The column statistics pass also yields the bias gradients (column sums of dG).
#include <stdlib.h>
#include <string.h>

#include "decoder.h"
#include "umma.cuh"
#include "wgrad_tc.h"

namespace t2 {

namespace {

constexpr int kTM = 128, kTN = 256;                  // tile: gate rows x feature rows
constexpr int kABytes = 2 * kTM * 128;               // [hi | lo] planes of 128 rows x 128 B = 32 KB
constexpr int kBBytes = 2 * kTN * 128;               // 64 KB
constexpr int kStageB = kABytes + kBBytes;           // 96 KB
constexpr int kWgStages = 2;
constexpr int kWgThreads = 384;                      // warp 0: producer; warpgroups 1 / 2: MMA + epilogue
constexpr int kStatSplit = kWgStatSplit;

// ---- column statistics of dG (rows x 4096): max |.| and sum per column ---------------------------------
__global__ void __launch_bounds__(256) wg_colstats_kernel(const float* __restrict__ x, long rows, int C, float* __restrict__ part) {
  __shared__ float rm[8][33], rs[8][33];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const long per = (rows + kStatSplit - 1) / kStatSplit;
  const long r0 = blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
  float mx = 0.f, sm = 0.f;
  if (c < C) for (long r = r0 + rg; r < r1; r += 8) {
    const float v = x[r * C + c];
    mx = fmaxf(mx, fabsf(v));
    sm += v;
  }
  rm[rg][cl] = mx; rs[rg][cl] = sm;
  __syncthreads();
  if (rg == 0 && c < C) {
    for (int i = 1; i < 8; ++i) { mx = fmaxf(mx, rm[i][cl]); sm += rs[i][cl]; }
    part[((long)blockIdx.y * 2 + 0) * C + c] = mx;
    part[((long)blockIdx.y * 2 + 1) * C + c] = sm;
  }
}
__global__ void wg_colstats_finalize_kernel(const float* __restrict__ part, int C, float* __restrict__ scale, float* __restrict__ inv_scale,
                                            float* __restrict__ colsum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mx = 0.f;
  double sm = 0.0;
  for (int i = 0; i < kStatSplit; ++i) { mx = fmaxf(mx, part[((long)i * 2) * C + c]); sm += (double)part[((long)i * 2 + 1) * C + c]; }
  int e = 0;
  if (mx > 0.f && mx < 3.0e38f) frexpf(mx, &e);
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  scale[c] = ldexpf(1.f, -e);
  inv_scale[c] = ldexpf(1.f, e);
  colsum[c] = (float)sm;
}

// ---- fp32 rows (chunk t = rows [t*B, t*B + B)) x C columns  ->  transposed operand images -----------------------
// image of chunk t: C / TR tiles, each [hi plane TR x 128 B | lo plane], element (row = c % TR, k = b) = src[t*B+b][c] * scale[c]
__global__ void __launch_bounds__(256) wg_transpose_img_kernel(const float* __restrict__ src, long ld, long row0, long rows_total,
                                                               int chunk_rows, int slices, int C, int TR, const float* __restrict__ scale,
                                                               uint8_t* __restrict__ img) {
  // group g = source rows [row0 + g * chunk_rows, + chunk_rows) as `slices` chunks of 64 rows: chunk t = slice t % slices
  // of group t / slices (chunk_rows <= 64 * slices; the remaining k and rows outside [0, rows_total) are zero); columns
  // >= C of the last tile are zero rows
  __shared__ float tile[64][65];
  const int c0 = blockIdx.x * 64, t = blockIdx.y, tid = threadIdx.x;
  const int g = t / slices, b0 = (t - g * slices) * 64;
  for (int i = tid; i < 64 * 64; i += 256) {
    const int b = i >> 6, cc = i & 63;
    const long r = row0 + (long)g * chunk_rows + b0 + b;
    tile[b][cc] = (b0 + b < chunk_rows && r >= 0 && r < rows_total && c0 + cc < C) ? src[r * ld + c0 + cc] : 0.f;
  }
  __syncthreads();
  const int ntile = (C + TR - 1) / TR;
  for (int i = tid; i < 64 * 8; i += 256) {
    const int cc = i >> 3, k8 = i & 7;
    const int c = c0 + cc, r = c % TR, q = c / TR;
    if (q >= ntile) continue;
    const float sc = (scale && c < C) ? scale[c] : 1.f;
    __align__(16) __half hh[8];
    __align__(16) __half ll[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split_fp16(tile[k8 * 8 + e][cc] * sc, hh[e], ll[e]);
    uint8_t* plane = img + ((size_t)t * ntile + q) * (size_t)(2 * TR * 128);
    const uint32_t off = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((k8 ^ (r & 7)) * 16));
    *reinterpret_cast<uint4*>(plane + off) = *reinterpret_cast<const uint4*>(hh);
    *reinterpret_cast<uint4*>(plane + (size_t)TR * 128 + off) = *reinterpret_cast<const uint4*>(ll);
  }
}

// ---- the GEMM ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_wait(uint64_t* bar, uint32_t parity) {
  const unsigned long long t0 = clock64();
  while (!ptx::mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > (1ull << 33)) __trap();
  }
}

// Jobs: the CTA table as a function of blockIdx.x (WgDecJobs, WgConvJobs)
template <class Jobs>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const Jobs jobs) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const WgJob job = jobs((int)blockIdx.x);
  uint8_t* stage0 = smem_raw;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + kWgStages * kStageB);
  uint64_t* full = bars; uint64_t* empty = bars + kWgStages;
  if (tid == 0) {
    for (int s = 0; s < kWgStages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 2); }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      const uint64_t pol = ptx::policy_evict_last();     // tiles are shared by the concurrently resident CTAs (job order)
      uint32_t s = 0, ph = 0;
      for (int i = 0; i < job.nchunks; ++i) {
        wg_wait(&empty[s], ph ^ 1);
        ptx::mbar_arrive_expect_tx(&full[s], kStageB);
        uint8_t* st = stage0 + (size_t)s * kStageB;
        ptx::bulk_g2s_hint(st, job.a + (size_t)i * job.a_stride, kABytes, &full[s], pol);
        ptx::bulk_g2s_hint(st + kABytes, job.b + (size_t)i * job.b_stride, kBBytes, &full[s], pol);
        if (++s == kWgStages) { s = 0; ph ^= 1; }
      }
    }
    __syncwarp();
  } else if (tid >= 128) {
    // warpgroup 1 / 2: gate rows [64 wg, 64 wg + 64) x all 256 feature columns (two 64 x 128 accumulators)
    const int wg = (tid >> 7) - 1, wt = tid & 127;
    float d0[64], d1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
    ptx::wg_fence_regs<64>(d0);
    ptx::wg_fence_regs<64>(d1);
    uint32_t s = 0, ph = 0;
    for (int i = 0; i < job.nchunks; ++i) {
      wg_wait(&full[s], ph);
      const uint32_t a_hi = ptx::smem_u32(stage0 + (size_t)s * kStageB) + (uint32_t)wg * (64 * 128), a_lo = a_hi + kTM * 128;
      const uint32_t b_hi = ptx::smem_u32(stage0 + (size_t)s * kStageB) + kABytes, b_lo = b_hi + kTN * 128;
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < kChunkK / 16; ++kk) {
        const uint64_t dah = ptx::make_sw128_desc(a_hi + kk * 32), dal = ptx::make_sw128_desc(a_lo + kk * 32);
        const uint64_t dbh0 = ptx::make_sw128_desc(b_hi + kk * 32), dbh1 = ptx::make_sw128_desc(b_hi + 128 * 128 + kk * 32);
        const uint64_t dbl0 = ptx::make_sw128_desc(b_lo + kk * 32), dbl1 = ptx::make_sw128_desc(b_lo + 128 * 128 + kk * 32);
        ptx::wgmma_f16<128>(d0, dah, dbh0);
        ptx::wgmma_f16<128>(d1, dah, dbh1);
        ptx::wgmma_f16<128>(d0, dah, dbl0);
        ptx::wgmma_f16<128>(d1, dah, dbl1);
        ptx::wgmma_f16<128>(d0, dal, dbh0);
        ptx::wgmma_f16<128>(d1, dal, dbh1);
      }
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_fence_regs<64>(d0);
      ptx::wg_fence_regs<64>(d1);
      if (wt == 0) ptx::mbar_arrive(&empty[s]);          // this warpgroup's MMAs have read the stage
      if (++s == kWgStages) { s = 0; ph ^= 1; }
    }
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int row = wg * 64 + ptx::wg_frag_row(i, wt), col = ptx::wg_frag_col(i, wt);
      const float sc = job.inv_scale[row];
      float* out = job.out + (size_t)row * job.ldo + col;
      *reinterpret_cast<float2*>(out) = make_float2(d0[i] * sc, d0[i + 1] * sc);
      *reinterpret_cast<float2*>(out + 128) = make_float2(d1[i] * sc, d1[i + 1] * sc);
    }
  }
}

// partial sums (nsplit, 4096, ldc) -> the parameter gradients: columns [0, c_ih) -> W_ih (4096 x c_ih), the rest -> W_hh (4096 x 1024)
__global__ void wg_reduce_kernel(const float* __restrict__ part, int nsplit, int ldc, int c_ih, float* __restrict__ g_ih,
                                 float* __restrict__ g_hh) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)4096 * ldc) return;
  const int c = (int)(i % ldc); const long r = i / ldc;
  float s = 0.f;
  for (int k = 0; k < nsplit; ++k) s += part[(long)k * 4096 * ldc + i];
  if (c < c_ih) { if (g_ih) g_ih[r * c_ih + c] = s; }
  else if (g_hh) g_hh[r * 1024 + (c - c_ih)] = s;
}

template <class Jobs>
int wg_launch(const Jobs& jobs, int n, cudaStream_t s) {
  const size_t smem = (size_t)kWgStages * kStageB + 256;
  T2_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<Jobs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  wgrad_tc_kernel<Jobs><<<n, kWgThreads, smem, s>>>(jobs);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

// The CTAs of the decoder LSTM weight gradients, in launch order: LSTM l, K split sp, gate tile i, feature tile (of the
// LSTM's concatenated input, group by group).  This order is L2 locality: all tiles of one K split (one 100-step window
// of the images) run together, gate tile outer, feature tile inner, so concurrently resident CTAs share their A and B
// tiles (ncu: 25.8 GB of DRAM reads for 2.2 GB of operands in the gate-tile-inner order).
struct WgDecJobs {
  struct Grp { const uint8_t* img; int ntile; int t0; };   // feature group: image, 256-row tiles per chunk, first chunk
  Grp grp[2][3];
  const uint8_t* img_a[2];
  float* part[2];
  const float* inv[2];
  int T, seg, nsplit;      // T: K chunks (decoder steps x 64-row chunks per step)
  __device__ WgJob operator()(int idx) const {
    const int n0 = nsplit * (4096 / kTM) * (1792 / kTN);      // CTAs of the attention LSTM
    const int l = idx >= n0 ? 1 : 0;
    if (l) idx -= n0;
    const int ldc = l ? 2560 : 1792, ntf = ldc / kTN;
    int jt = idx % ntf;
    const int col = jt * kTN;
    idx /= ntf;
    const int i = idx % (4096 / kTM), sp = idx / (4096 / kTM);
    int g = 0;
    while (jt >= grp[l][g].ntile) jt -= grp[l][g++].ntile;
    const Grp gr = grp[l][g];
    const int c0 = sp * seg;
    WgJob j;
    j.a_stride = (uint32_t)(4096 / kTM) * kABytes; j.b_stride = (uint32_t)gr.ntile * kBBytes;
    j.a = img_a[l] + (size_t)c0 * j.a_stride + (size_t)i * kABytes;
    j.b = gr.img + (size_t)(c0 + gr.t0) * j.b_stride + (size_t)jt * kBBytes;
    j.nchunks = min(T - c0, seg);
    j.out = part[l] + ((size_t)sp * 4096 + (size_t)i * kTM) * ldc + col;
    j.ldo = ldc;
    j.inv_scale = inv[l] + i * kTM;
    return j;
  }
};

}  // namespace

// K chunks of 64 rows per decoder step: the B rows of a step as ceil(B / 64) zero-padded chunks
static int wgrad_step_chunks(int B) { return (B + 63) / 64; }

void wgrad_tc_layout(Carve& c, int B, int T, WgradWs* w) {
  const int S = wgrad_step_chunks(B), nch = T * S;
  const int seg = wgrad_seg(nch), nsplit = (nch + seg - 1) / seg;
  for (int l = 0; l < 2; ++l) w->img_a[l] = c.take<uint8_t>((size_t)nch * 4096 * 256, 1024);
  w->img_x2 = c.take<uint8_t>((size_t)nch * 256 * 256, 1024);
  w->img_ctx = c.take<uint8_t>((size_t)(T + 1) * S * 1024 * 256, 1024);
  w->img_ha = c.take<uint8_t>((size_t)(T + 1) * S * 1024 * 256, 1024);
  w->img_hd = c.take<uint8_t>((size_t)(T + 1) * S * 1024 * 256, 1024);
  w->part = c.take<float>((size_t)nsplit * 4096 * (1792 + 2560), 1024);
  w->stat = c.take<float>((size_t)kStatSplit * 2 * 4096, 1024);
  w->scale = c.take<float>(4096, 1024);
  for (int l = 0; l < 2; ++l) w->inv[l] = c.take<float>(4096, 1024);
  w->colsum = c.take<float>(4096, 1024);
}

// dga / dgd: (T, B, 4096) fp32; x2 (T, B, 256); stash slots ctx (T+1, B, 512), ha / hd (T+1, B, 1024).
int wgrad_tc_run(T2Model* m, int B, int T, const float* dga, const float* dgd, const float* x2, const DecoderStash& st,
                 float* const* G, const WgradWs& w, cudaStream_t s) {
  (void)m;
  const int S = wgrad_step_chunks(B), nch = T * S;
  const int seg = wgrad_seg(nch), nsplit = (nch + seg - 1) / seg;
  const long rows = (long)T * B;
  const float* dG[2] = {dga, dgd};
  const int bias_idx[2][2] = {{W_ARNN_BIH, W_ARNN_BHH}, {W_DRNN_BIH, W_DRNN_BHH}};
  for (int l = 0; l < 2; ++l) {
    wg_colstats_kernel<<<dim3(4096 / 32, kStatSplit), 256, 0, s>>>(dG[l], rows, 4096, w.stat);
    T2_LAUNCH_CHECK();
    wg_colstats_finalize_kernel<<<4096 / 128, 128, 0, s>>>(w.stat, 4096, w.scale, w.inv[l], w.colsum);
    T2_LAUNCH_CHECK();
    for (int k = 0; k < 2; ++k)
      if (G[bias_idx[l][k]]) T2_CUDA(cudaMemcpyAsync(G[bias_idx[l][k]], w.colsum, 4096 * 4, cudaMemcpyDeviceToDevice, s));
    wg_transpose_img_kernel<<<dim3(4096 / 64, nch), 256, 0, s>>>(dG[l], 4096, 0, rows, B, S, 4096, kTM, w.scale, w.img_a[l]);
    T2_LAUNCH_CHECK();
  }
  wg_transpose_img_kernel<<<dim3(256 / 64, nch), 256, 0, s>>>(x2, 256, 0, rows, B, S, 256, kTN, nullptr, w.img_x2);
  T2_LAUNCH_CHECK();
  wg_transpose_img_kernel<<<dim3(512 / 64, (T + 1) * S), 256, 0, s>>>(st.ctx, 512, 0, rows + B, B, S, 512, kTN, nullptr, w.img_ctx);
  T2_LAUNCH_CHECK();
  wg_transpose_img_kernel<<<dim3(1024 / 64, (T + 1) * S), 256, 0, s>>>(st.ha, 1024, 0, rows + B, B, S, 1024, kTN, nullptr, w.img_ha);
  T2_LAUNCH_CHECK();
  wg_transpose_img_kernel<<<dim3(1024 / 64, (T + 1) * S), 256, 0, s>>>(st.hd, 1024, 0, rows + B, B, S, 1024, kTN, nullptr, w.img_hd);
  T2_LAUNCH_CHECK();
  WgDecJobs jobs;
  jobs.grp[0][0] = {w.img_x2, 1, 0}; jobs.grp[0][1] = {w.img_ctx, 2, 0}; jobs.grp[0][2] = {w.img_ha, 4, 0};   // [x2_t | ctx_(t-1) | ah_(t-1)]   model.py:352
  jobs.grp[1][0] = {w.img_ha, 4, S}; jobs.grp[1][1] = {w.img_ctx, 2, S}; jobs.grp[1][2] = {w.img_hd, 4, 0};   // [ah_t | ctx_t | dh_(t-1)]       model.py:366-367
  float* part_l[2] = {w.part, w.part + (size_t)nsplit * 4096 * 1792};
  for (int l = 0; l < 2; ++l) { jobs.img_a[l] = w.img_a[l]; jobs.part[l] = part_l[l]; jobs.inv[l] = w.inv[l]; }
  jobs.T = nch; jobs.seg = seg; jobs.nsplit = nsplit;
  T2_TRY(wg_launch(jobs, nsplit * (4096 / kTM) * ((1792 + 2560) / kTN), s));
  {
    const long n = (long)4096 * 1792;
    wg_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(part_l[0], nsplit, 1792, 768, G[W_ARNN_WIH], G[W_ARNN_WHH]);
    T2_LAUNCH_CHECK();
  }
  {
    const long n = (long)4096 * 2560;
    wg_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(part_l[1], nsplit, 2560, 1536, G[W_DRNN_WIH], G[W_DRNN_WHH]);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}


// ---- generic entry points (also used by the conv-stack weight gradients in train_layers.cu) ------------------------
int wg_run_jobs(const WgConvJobs& jobs, cudaStream_t s) { return wg_launch(jobs, jobs.count(), s); }
size_t wg_colstats_ws_bytes(int C) { return (size_t)kStatSplit * 2 * C * sizeof(float); }
int wg_colstats(const float* x, long rows, int C, float* stat_ws, float* scale, float* inv_scale, float* colsum, cudaStream_t s) {
  wg_colstats_kernel<<<dim3((C + 31) / 32, kStatSplit), 256, 0, s>>>(x, rows, C, stat_ws);
  T2_LAUNCH_CHECK();
  wg_colstats_finalize_kernel<<<(C + 127) / 128, 128, 0, s>>>(stat_ws, C, scale, inv_scale, colsum);
  T2_LAUNCH_CHECK();
  return T2_OK;
}
int wg_transpose_images(const float* src, long ld, long row0, long rows_total, int chunk_rows, int nchunks, int C, int TR,
                        const float* scale, uint8_t* img, cudaStream_t s) {
  const int ntile = (C + TR - 1) / TR;
  wg_transpose_img_kernel<<<dim3(ntile * TR / 64, nchunks), 256, 0, s>>>(src, ld, row0, rows_total, chunk_rows, 1, C, TR, scale, img);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
