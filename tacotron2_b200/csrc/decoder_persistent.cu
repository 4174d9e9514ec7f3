// T2_IMPL_PERSISTENT: the whole autoregressive decoder loop (model.py:381-454) as ONE persistent
// cooperative sm_90a kernel.
//
//   * 128 CTAs (one per SM), 512 threads each.  CTA c owns hidden units [8c, 8c+8) of BOTH
//     LSTM cells (attention_rnn, decoder_rnn): their cell state lives in registers for the whole loop,
//     their gate pre-activations accumulate in a shared-memory fp32 tile across events.
//   * "activation driven" schedule: whenever a new activation block (x2, ah, ctx, dh, x1) is complete,
//     every CTA streams it ONCE through a shared-memory ring (bulk async copies on the TMA engine)
//     together with the slices of every weight matrix that consumes it, and three warpgroups issue wgmma:
//        x2_t  -> att gates += W_ih^a[:, :256] x2                          -> ah_t, ac_t
//        ah_t  -> dec gates += W_ih^d[:, :1024] ah ; att gates(t+1) += W_hh^a ah ; q = W_q ah
//        ctx_t -> dec gates += W_ih^d[:, 1024:] ctx ; att gates(t+1) += W_ih^a[:, 256:] ctx ;
//                 proj += W_P[:, 1024:] ctx                                 -> dh_t, dc_t
//        dh_t  -> proj += W_P[:, :1024] dh ; dec gates(t+1) += W_hh^d dh   -> mel_t, gate_t, x1
//        x1    -> x2_(t+1) = relu(W_2 x1) * mask
//     W_P stacks linear_projection, gate_layer and (W_1 . W_proj), so the first prenet layer of the
//     NEXT step is computed from [dh; ctx] directly (model.py:97-100, 373-378, 449).
//   * fp32-grade arithmetic on fp16 tensor cores: every operand is split x = hi + lo (two fp16).  The
//     activation chunk image is [X_hi rows 0-63 | X_lo rows 64-127]; the weight rows of all consumers of
//     an event are concatenated as [W_hi ; W_lo] per consumer.  All four partial products (hi.hi, lo.hi,
//     hi.lo, lo.lo) are kept.  Warpgroup 1 + c owns consumer c (<= 32 rows) and takes its [W_hi ; W_lo]
//     rows as ONE wide B operand (N = 2n), so a 16-wide K step is two wgmma m64n(2n)k16 instead of four
//     m64nnk16, and each X plane is read once per consumer and K step:
//        D[64 x 2n] += X_hi . [W_hi ; W_lo]^T + X_lo . [W_hi ; W_lo]^T
//     At the end of the event the warpgroup adds the W_hi and W_lo column halves of D and adds the sum to
//     the shared-memory accumulator tile.  Accumulators are always accumulated into and zeroed by the
//     epilogue that consumed them.
//   * location-sensitive attention (model.py:43-86): location conv + dense are fused into one 62-tap
//     filter bank evaluated as a tensor-core GEMM over an im2col image of the previous / cumulative
//     weights (kept in shared memory across steps); energies, softmax and context per batch row on a
//     CTA pair with warp-shuffle reductions.
//   * events are separated by a grid-wide barrier or by producer-scoped counters (monotonic global counters:
//     fence.acq_rel + relaxed red to arrive, relaxed polls + one fence to wait).
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "decoder.h"
#include "gemm_f32.cuh"
#include "umma.cuh"

namespace t2 {

namespace {

constexpr int kG = 128;               // CTAs
constexpr int kThreads = 512;
constexpr int kStages = 4;             // ring stages of the helper kernels (self test, backward GEMMs)
constexpr int kMaxStages = 4;          // the decoder kernel runs 4 stages up to T_enc = 896, else 3
                                       // (T2_STAGES = 3 forces the 3-stage ring)
constexpr int kRows = 64;             // batch rows per launch (zero padded)
constexpr int kXChunkBytes = 2 * kRows * kChunkK * 2;    // [hi 64 rows | lo 64 rows] x 64 k fp16 = 16 KiB
// accumulator columns (shared memory, fp32 [64 batch rows][kAccPitch]): att 0-31, dec 32-63, shared slot 64-79
constexpr int kColA = 0, kColD = 32, kColS = 64;
constexpr int kHiCols = 80;                               // max weight rows of one event (hi)
constexpr int kAccPitch = 84;                             // floats per accumulator row (80 + 4: fewer bank conflicts)
constexpr int kAccBytes = kRows * kAccPitch * 4;
constexpr int kMmaWgs = 3;                                // warpgroups 1-3 issue the MMAs of an event (one piece each)
constexpr int kAttRound = 64;                             // encoder positions per attention pa GEMM
constexpr int kAttPlane = kAttRound * 128;                // one fp16 plane of the im2col image (64 positions x 64 taps)
constexpr int kPaPitch = kAttRound + 4;                   // floats per attention dim of the pa tile
constexpr int kPaBytes = kAtt * kPaPitch * 4;
constexpr int kWStageMax = 2 * kHiCols * kChunkK * 2;    // hi + lo planes of up to 80 weight rows = 20 KiB
constexpr int kStageBytes = kXChunkBytes + kWStageMax;   // 36 KiB
constexpr int kNumEvents = 5;         // x2, ah, ctx, dh, x1
constexpr int kPCols = 344;           // 80 mel + 1 gate + 256 x1 + 7 pad
constexpr int kQCta0 = 0, kQCtas = 16, kX2Cta0 = 16, kX2Ctas = 32, kPCta0 = 48, kPCtas = 43;
constexpr int kWeffBytes = kAtt * kChunkK * 2 * 2;        // fused location filter image (hi+lo) = 32 KiB
constexpr unsigned long long kWatchdogCycles = 1ull << 32;   // ~2 s

struct EventPlan {
  uint32_t w_off;       // byte offset of this CTA's first chunk in the W image buffer
  uint32_t w_bytes;     // W bytes per chunk = 2 x nrows x 128
  int32_t nrows;        // hi weight rows of all consumers (MMA N = 2 x nrows); 0 = this CTA skips the event
  int32_t col0;         // accumulator column of the first consumer
  int32_t ncons;
  int32_t n[3];         // rows per consumer (packing only)
  int32_t chunks;       // K chunks of this event (bounds the weight prefetch)
};
struct CtaPlan {
  EventPlan ev[kNumEvents];
};

struct BwdCta {          // one CTA of a backward skinny GEMM: a tile of output columns x a range of K chunks
  EventPlan ep;
  int32_t chunk0, nchunks;   // K chunks (64 gate rows each) of this CTA
  int32_t col0, split;       // first output column, index of the K split (partials)
};

struct PersistentPack {
  uint8_t* wimg = nullptr; size_t wimg_bytes = 0;
  CtaPlan* plans = nullptr;           // device, kG entries
  float* wp_all = nullptr;            // (344, 1536) fp32: proj | gate | W1.Wproj | zero pad
  float* bias_p = nullptr;            // (344): proj bias | gate bias | W1.b_proj | 0
  float* bias_a = nullptr;            // (kG, 32) att LSTM bias in accumulator column order
  float* bias_d = nullptr;            // (kG, 32)
  int32_t* rows = nullptr;            // row tables for packing
  float* weff = nullptr;              // (128, 64) fp32 fused location filter W_ld . W_loc (62 taps + 2 zero)
  uint8_t* weff_img = nullptr;        // its split-fp16 operand image (32 KiB)
  // backward skinny GEMMs (training): CTA plans of the decoder (0) and attention (1) LSTM (their weight images are packed
  // into the backward workspace by every call)
  BwdCta* bwd_plans[2] = {nullptr, nullptr};
};
std::vector<BwdCta> bwd_gemm_plans(int which);   // the CTA plans of a backward skinny GEMM

// ---------------------------------------------------------------------------------------------
// packing kernels (model create time)
// ---------------------------------------------------------------------------------------------
// W1P = W1 (256x80) . Wproj (80x1536), b1p = W1 . bproj           (fusing model.py:375-376 into :98)
__global__ void fuse_prenet_proj_kernel(const float* __restrict__ w1, const float* __restrict__ wp,
                                        const float* __restrict__ bp, float* __restrict__ out_w,
                                        float* __restrict__ out_b) {
  const int r = blockIdx.x;                  // 0..255
  for (int c = threadIdx.x; c < kDRnn + kEnc; c += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < kMel; ++k) s = fmaf(w1[r * kMel + k], wp[(long)k * (kDRnn + kEnc) + c], s);
    out_w[(long)r * (kDRnn + kEnc) + c] = s;
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < kMel; ++k) s = fmaf(w1[r * kMel + k], bp[k], s);
    out_b[r] = s;
  }
}

// Weff[d][ch*31+k] = sum_c W_ld[d][c] * W_loc[c][ch][k]: location conv (model.py:23) and location dense
// (model.py:24-25) are both linear, so they fuse into one 62-tap filter bank per attention dimension.
__global__ void fuse_location_kernel(const float* __restrict__ wld, const float* __restrict__ wloc,
                                     float* __restrict__ weff) {
  const int d = blockIdx.x, kk = threadIdx.x;      // 128 x 64
  float s = 0.f;
  if (kk < 2 * kLocK) {
    const int ch = kk / kLocK, k = kk - ch * kLocK;
    for (int c = 0; c < kLocF; ++c) s = fmaf(wld[d * kLocF + c], wloc[(c * 2 + ch) * kLocK + k], s);
  }
  weff[d * kChunkK + kk] = s;
}

// (N x K) fp32 row-major -> K/64 chunks of [hi plane | lo plane] (N rows each) in the canonical layout
__global__ void pack_rows_image_kernel(const float* __restrict__ W, int N, int K, uint8_t* __restrict__ wimg) {
  const int chunk = blockIdx.x;
  __half* hi = reinterpret_cast<__half*>(wimg + (size_t)chunk * N * 256);
  __half* lo = hi + N * 64;
  for (int i = threadIdx.x; i < N * 64; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    __half h, l;
    split_fp16(W[(long)r * K + chunk * 64 + k], h, l);
    const uint32_t e = img_elem_offset(r, k);
    hi[e] = h; lo[e] = l;
  }
}

// one consumer of one event: for CTA blockIdx.y, chunk blockIdx.x: rows rows_tab[cta*32 + i] (-1 = zero
// row) x 64 columns starting at kcol0 + chunk*64 go to rows [roff, roff+n) of the chunk's hi and lo planes
// (each plane holds the rows of ALL consumers of the event, concatenated).
__global__ void pack_consumer_kernel(const float* __restrict__ src, int ld, int kcol0,
                                     const int32_t* __restrict__ rows_tab, const CtaPlan* __restrict__ plans,
                                     int ev, int cons, uint8_t* __restrict__ wimg) {
  const int cta = blockIdx.y, chunk = blockIdx.x;
  const EventPlan& ep = plans[cta].ev[ev];
  if (cons >= ep.ncons) return;
  const int n = ep.n[cons];
  int roff = 0;                               // rows before this consumer: [hi | lo] of each earlier one
  for (int i = 0; i < cons; ++i) roff += 2 * ep.n[i];
  __half* img = reinterpret_cast<__half*>(wimg + ep.w_off + (size_t)chunk * ep.w_bytes);
  for (int i = threadIdx.x; i < n * 64; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    const int srow = rows_tab[cta * 32 + r];
    const float v = srow >= 0 ? src[(long)srow * ld + kcol0 + chunk * 64 + k] : 0.f;
    __half h, l;
    split_fp16(v, h, l);
    img[img_elem_offset(roff + r, k)] = h;
    img[img_elem_offset(roff + n + r, k)] = l;
  }
}

__global__ void pack_lstm_bias_kernel(const float* __restrict__ b_sum, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;     // cta*32 + col
  if (i >= kG * 32) return;
  const int cta = i >> 5, col = i & 31, ul = col >> 2, g = col & 3;
  out[i] = b_sum[g * 1024 + cta * 8 + ul];
}

// fp32 rows (n_rows x K, ld) -> activation images: chunks x [hi rows 0-63 | lo rows 64-127] x 64 k
__global__ void rows_to_image_kernel(const float* __restrict__ src, long ld, int n_rows, int K,
                                     long src_block_stride, uint8_t* __restrict__ dst, long dst_block_stride) {
  const float* s = src + (long)blockIdx.y * src_block_stride;
  uint8_t* d = dst + (long)blockIdx.y * dst_block_stride;
  const int chunk = blockIdx.x;
  __half* hi = reinterpret_cast<__half*>(d + (long)chunk * kXChunkBytes);
  __half* lo = hi + kRows * kChunkK;
  for (int i = threadIdx.x; i < kRows * kChunkK; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    const int kk = chunk * kChunkK + k;
    const float v = (r < n_rows && kk < K) ? s[(long)r * ld + kk] : 0.f;
    __half h, l;
    split_fp16(v, h, l);
    const uint32_t e = img_elem_offset(r, k);
    hi[e] = h; lo[e] = l;
  }
}

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void watchdog_trap(DecoderCtrl* ctrl, int code) {
  if (ctrl) ctrl->error = code;
  __threadfence_system();
  __trap();
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, DecoderCtrl* ctrl, int code) {
  if (ptx::mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = clock64();
  while (!ptx::mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > kWatchdogCycles) watchdog_trap(ctrl, code);
  }
}

// One thread of a CTA publishes the CTA's stores (ordered before it by __syncthreads) and bumps a counter: a single
// gpu-scope fence followed by a relaxed reduction (fence + relaxed atomic = release; __threadfence() followed by
// red.release paid for two fences).  The waiting side polls with relaxed loads and fences once after the value
// arrived (an acquire load per poll iteration costs a fence per iteration).
__device__ __forceinline__ void arrive_release(unsigned int* cnt) {
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(cnt) : "memory");
}
__device__ __forceinline__ void poll_acquire(unsigned int* cnt, unsigned int target, DecoderCtrl* ctrl, int code) {
  const unsigned long long t0 = clock64();
  while (true) {
    unsigned int c;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(c) : "l"(cnt) : "memory");
    if ((int)(c - target) >= 0) break;
    if (clock64() - t0 > kWatchdogCycles) watchdog_trap(ctrl, code);
  }
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
}

// grid-wide barrier: one monotonically increasing arrival counter; arrive = arrive_release, wait = poll_acquire
// until the counter reaches this barrier's target (no reset / generation hop).  Also orders the generic-proxy
// stores of the epilogues before the async-proxy (bulk copy) reads of the next event.
__device__ __forceinline__ void grid_barrier(DecoderCtrl* ctrl, unsigned int& target) {
  ptx::fence_proxy_async();
  __syncthreads();
  target += gridDim.x;
  if (threadIdx.x == 0) {
    arrive_release(&ctrl->bar_count);
    poll_acquire(&ctrl->bar_count, target, ctrl, 100);
  }
  __syncthreads();
  ptx::fence_proxy_async();
}

// split-phase form of the flat barrier: arrive as soon as this CTA's contribution is written, do work that
// does not depend on the other CTAs, then wait
__device__ __forceinline__ void grid_arrive(DecoderCtrl* ctrl, unsigned int& target) {
  ptx::fence_proxy_async();
  __syncthreads();
  target += gridDim.x;
  if (threadIdx.x == 0) {
    arrive_release(&ctrl->bar_count);
  }
}
__device__ __forceinline__ void grid_wait(DecoderCtrl* ctrl, unsigned int target) {
  if (threadIdx.x == 0) {
    poll_acquire(&ctrl->bar_count, target, ctrl, 101);
  }
  __syncthreads();
  ptx::fence_proxy_async();
}

// producer-scoped hand-over: the producers of a block signal a monotonic counter once their stores are done, the
// consumers wait until it reaches (#producers x step).  Same fences as the grid barrier on both sides.
constexpr unsigned int kStopFlag = 1u << 24;    // counters count arrivals in bits 0-23 (32 x 524k steps), bits 24+ = "stop"
__device__ __forceinline__ void signal_counter(unsigned int* cnt, unsigned int inc) {
  ptx::fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
    asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(cnt), "r"(inc) : "memory");
  }
}
// returns true when a producer attached the stop flag
__device__ __forceinline__ bool wait_counter(unsigned int* cnt, unsigned int target, int* s_flag, DecoderCtrl* ctrl, int code) {
  if (threadIdx.x == 0) {
    const unsigned long long t0 = clock64();
    unsigned int c;
    while (true) {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(c) : "l"(cnt) : "memory");
      if ((c & (kStopFlag - 1u)) >= target) break;
      if (clock64() - t0 > kWatchdogCycles) watchdog_trap(ctrl, code);
    }
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
    *s_flag = (int)(c >> 24);
  }
  __syncthreads();
  ptx::fence_proxy_async();
  return *s_flag != 0;
}

__device__ __forceinline__ float sigmoid_exact(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 2.f * sigmoid_fast(2.f * x) - 1.f; }
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct Ring {
  uint8_t* stage0;    // kStages buffers of kStageBytes each
  __device__ __forceinline__ uint8_t* stage(uint32_t s) const { return stage0 + s * kStageBytes; }
  uint64_t* full;     // [kStages]
  uint64_t* empty;    // [kStages], released once by each MMA warpgroup
  uint32_t p_stage, p_phase;   // producer cursor (thread 0 of warp 0)
  uint32_t c_stage, c_phase;   // consumer cursor (threads of the MMA warpgroups 1-3)
  uint64_t pol_x, pol_w;       // L2 eviction policies of the activation / weight streams
  uint32_t pre;                // stages whose weight chunk was already issued for the upcoming event
  uint32_t ns;                 // number of stages
};

// Dynamic shared memory of the persistent decoder for (T_enc, ring stages): the kernel carves it and the host sizes
// the launch from it, which decides the ring depth and the longest T_enc.  The regions are packed in this order.
struct PersistentSmem {
  uint8_t* stage0;                 // ring stages
  uint8_t* weff;                   // fused location filter image
  float* acc;                      // event accumulators
  uint64_t* bars;                  // 16 slots: full[kMaxStages] | empty[kMaxStages]
  int* live;                       // [0] live rows, [1] stop flag broadcast of wait_counter
  float *bias_a, *bias_d, *v, *q;
  float* red;                      // unused; kept so the regions after it stay where they are
  uint32_t* mask;                  // prenet keep bits of step t+1 (8 per row)
  float* bias_p;                   // bias of this CTA's 8 projection columns
  long long* prof;                 // phase profile, accumulated on chip
  float *pad0, *pad1;              // previous | cumulative attention weights (padded)
  float* e;                        // [ntiles * 128] attention weights
  float* ep;                       // [4][ntiles * 128] energy partial sums
};
__host__ __device__ __forceinline__ void persistent_smem_layout(Carve& c, int T, int nstages, PersistentSmem* s) {
  const int tpp = (T + kLocK - 1 + 3) & ~3, ntiles = (T + 127) >> 7;
  s->stage0 = c.take<uint8_t>((size_t)nstages * kStageBytes, 1);
  s->weff = c.take<uint8_t>(kWeffBytes, 1);
  s->acc = c.take<float>(kAccBytes / 4, 1);
  s->bars = c.take<uint64_t>(16, 1);
  s->live = c.take<int>(4, 1);
  s->bias_a = c.take<float>(32, 1); s->bias_d = c.take<float>(32, 1);
  s->v = c.take<float>(kAtt, 1); s->q = c.take<float>(kAtt, 1);
  s->red = c.take<float>(32, 1);
  s->mask = c.take<uint32_t>(kRows, 1);
  s->bias_p = c.take<float>(8, 1);
  s->prof = c.take<long long>(24, 1);
  s->pad0 = c.take<float>(tpp, 1); s->pad1 = c.take<float>(tpp, 1);
  s->e = c.take<float>((size_t)ntiles * 128, 1);
  s->ep = c.take<float>((size_t)4 * ntiles * 128, 1);
}

// Dynamic shared memory of the self test and the backward GEMMs: ring stages, barriers, then the accumulator tile
struct GemmSmem { uint8_t* stage0; uint64_t* bars; float* acc; };
__host__ __device__ __forceinline__ void gemm_smem_layout(Carve& c, GemmSmem* s) {
  s->stage0 = c.take<uint8_t>((size_t)kStages * kStageBytes, 1);
  s->bars = c.take<uint64_t>(16, 1);
  s->acc = c.take<float>(kAccBytes / 4, 1);      // [64][kAccPitch]
}
size_t gemm_smem_bytes() { Carve c(nullptr, 1); GemmSmem s; gemm_smem_layout(c, &s); return c.bytes(); }

// Weight chunks do not depend on the grid barrier that separates two events (only the activation does):
// the producer arms the first kStages stages of the NEXT event and issues their weight copies right after
// the current event's last chunk, so their L2 / HBM latency overlaps the epilogue and the barrier.
__device__ __forceinline__ void prefetch_weights(Ring& rg, const EventPlan& nx, const uint8_t* w_img,
                                                 DecoderCtrl* ctrl) {
  uint32_t s = rg.p_stage, ph = rg.p_phase;
  const uint32_t n = min(rg.ns, (uint32_t)nx.chunks);
  for (uint32_t i = 0; i < n; ++i) {
    mbar_wait(&rg.empty[s], ph ^ 1, ctrl, 205);
    ptx::mbar_arrive_expect_tx(&rg.full[s], kXChunkBytes + nx.w_bytes);
    ptx::bulk_g2s_hint(rg.stage(s) + kXChunkBytes, w_img + nx.w_off + (size_t)i * nx.w_bytes, nx.w_bytes,
                       &rg.full[s], rg.pol_w);
    if (++s == rg.ns) { s = 0; ph ^= 1; }
  }
  rg.pre = n;
}

// How the three MMA warpgroups split an event.  Each consumer's rows sit in the stage as [n hi rows | n lo rows], so
// warpgroup 1 + c takes consumer c (n <= 32 rows) as ONE wgmma B operand of N = 2 n rows [W_hi; W_lo] and multiplies it
// with A = X_hi and A = X_lo: two wgmma per 16-wide K step, each reading its activation plane and the consumer's rows
// once (instead of four with separate hi / lo B operands, each re-reading an A plane).  N stays <= 64 (32 accumulator
// registers): the kernel runs at the 128-register limit of 512 threads, and a wider accumulator spills.
// all_widths = false: the consumer widths run_event<false> (decoder, backward GEMMs) is built for
inline bool event_plan_fits(const EventPlan& ep, bool all_widths) {
  if (ep.ncons < 1 || ep.ncons > kMmaWgs) return false;
  for (int c = 0; c < ep.ncons; ++c)
    if (ep.n[c] != 16 && ep.n[c] != 32 && !(all_widths && (ep.n[c] == 8 || ep.n[c] == 24))) return false;
  return true;
}
// `rows` output rows of one matrix as consumers that fit the warpgroups: 32, 32, rest (rows <= 80, a multiple of 8)
inline void plan_one_matrix(EventPlan& ep, int rows) {
  ep.ncons = 0; ep.nrows = rows;
  for (int r = rows; r > 0 && ep.ncons < 3; ) {
    const int n = ep.ncons < 2 && r >= 32 ? 32 : r;
    ep.n[ep.ncons++] = n; r -= n;
  }
  ep.w_bytes = (uint32_t)rows * 256;
}
// image rows of the hi and lo copies of row r (counted over all consumers) of a plan
__device__ __forceinline__ void plan_image_rows(const EventPlan& ep, int r, int& hi, int& lo) {
  int roff = 0;
  for (int c = 0; c < ep.ncons; ++c) {
    if (r < ep.n[c]) { hi = roff + r; lo = hi + ep.n[c]; return; }
    r -= ep.n[c]; roff += 2 * ep.n[c];
  }
  hi = lo = 0;
}

// One MMA warpgroup's consumer of an event: D (64 x 2n) = X_hi . B^T + X_lo . B^T over all `chunks` stages, where B is
// the consumer's 2n weight-image rows [W_hi; W_lo] from row w_row0 of each stage; then both column halves of D are
// added to the accumulator tile from column acol.  Each chunk's stage is released as soon as its MMAs are done: keeping
// a commit group in flight across chunks would hold every stage one chunk longer, i.e. make the ring one stage shallower
// for the producer, and the stream waits on L2 latency rather than on the tensor core (measured slower).
template <int N>
__device__ __forceinline__ void event_wg(Ring& rg, int chunks, uint32_t w_row0, float* s_acc, int acol, DecoderCtrl* ctrl) {
  const bool leader = (threadIdx.x & 127) == 0;
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  for (int i = 0; i < chunks; ++i) {
    mbar_wait(&rg.full[rg.c_stage], rg.c_phase, ctrl, 201);
    const uint32_t xs = ptx::smem_u32(rg.stage(rg.c_stage));
    const uint32_t ws = xs + kXChunkBytes + w_row0 * 128;
    ptx::wg_fence_regs<N / 2>(d);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < kChunkK / 16; ++kk) {
      const uint64_t b = ptx::make_sw128_desc(ws + kk * 32);
      ptx::wgmma_f16<N>(d, ptx::make_sw128_desc(xs + kk * 32), b);                  // X_hi
      ptx::wgmma_f16<N>(d, ptx::make_sw128_desc(xs + kRows * 128 + kk * 32), b);    // X_lo
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::wg_fence_regs<N / 2>(d);
    if (leader) ptx::mbar_arrive(&rg.empty[rg.c_stage]);
    if (++rg.c_stage == rg.ns) { rg.c_stage = 0; rg.c_phase ^= 1; }
  }
  const int wt = threadIdx.x & 127;
#pragma unroll
  for (int j = 0; j < N / 4; ++j)      // registers [0, N/4) hold the W_hi columns, [N/4, N/2) the W_lo ones
    s_acc[ptx::wg_frag_row(j, wt) * kAccPitch + acol + ptx::wg_frag_col(j, wt)] += d[j] + d[N / 4 + j];
}

// Streams `chunks` K-chunks of the activation image x_img plus this CTA's weight rows through the ring;
// warpgroups 1-3 issue the MMAs (one consumer each) and add their products to the accumulator tile s_acc.  Called by all threads;
// returns after the accumulators are complete.  Every MMA accumulates (the epilogues zero what they consume).
// The decoder's and the backward GEMMs' consumers have 32 or 16 rows (event_plan_fits(ep, false)); only the self test
// instantiates the 8- and 24-row consumers (kAllWidths): every width is a copy of the whole chunk loop, and the
// decoder kernel runs its code once per step, so each copy costs instruction-cache misses.
template <bool kAllWidths = false>
__device__ __forceinline__ void run_event(Ring& rg, const EventPlan& ep, const uint8_t* x_img,
                                          const uint8_t* w_img, int chunks, float* s_acc,
                                          DecoderCtrl* ctrl, const EventPlan* next,
                                          const unsigned int* ready = nullptr, unsigned int ready_target = 0) {
  // ready (16 counters, one per K chunk of the activation; null = the caller synchronised already): chunk i of x_img is
  // complete once ready[i] >= ready_target.  The activation blocks ah / dh are written in 8-column slices by 128 CTAs, i.e.
  // a 64-column chunk has 8 producers: instead of a 128-way barrier between the epilogue that writes a block and the event
  // that streams it, the bulk-copy producer fetches a chunk as soon as ITS 8 producers have arrived, so the stragglers'
  // skew and the arrival latency overlap with the streaming of the chunks that are already there.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (ep.nrows == 0) {                 // this CTA has no consumer of this activation
    if (threadIdx.x == 0 && next != nullptr && next->nrows != 0 && rg.pre == 0) prefetch_weights(rg, *next, w_img, ctrl);
    return;
  }
  if (warp == 0) {
    if (lane == 0) {
      int nready = ready ? 0 : chunks;     // chunks [0, nready) are known to be complete
      for (int i = 0; i < chunks; ++i) {
        uint8_t* st = rg.stage(rg.p_stage);
        if ((uint32_t)i >= rg.pre) {     // not armed / issued ahead of time
          mbar_wait(&rg.empty[rg.p_stage], rg.p_phase ^ 1, ctrl, 200);
          ptx::mbar_arrive_expect_tx(&rg.full[rg.p_stage], kXChunkBytes + ep.w_bytes);
          ptx::bulk_g2s_hint(st + kXChunkBytes, w_img + ep.w_off + (size_t)i * ep.w_bytes, ep.w_bytes,
                             &rg.full[rg.p_stage], rg.pol_w);
        }
        if (i >= nready) {               // all 16 counters in one round trip; take the leading run of complete chunks
          const unsigned long long t0 = clock64();
          while (true) {
            uint32_t c[16];
#pragma unroll
            for (int j = 0; j < 16; j += 4)
              asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                           : "=r"(c[j]), "=r"(c[j + 1]), "=r"(c[j + 2]), "=r"(c[j + 3]) : "l"(ready + j) : "memory");
            uint32_t mask = 0;
#pragma unroll
            for (int j = 0; j < 16; ++j) mask |= ((int)(c[j] - ready_target) >= 0 ? 1u : 0u) << j;
            const int run = __ffs((int)~(mask >> i)) - 1;          // complete chunks starting at i
            if (run > 0) { nready = min(chunks, i + run); break; }
            if (clock64() - t0 > kWatchdogCycles) watchdog_trap(ctrl, 206);
          }
          asm volatile("fence.acq_rel.gpu;" ::: "memory");
          ptx::fence_proxy_async();
        }
        ptx::bulk_g2s_hint(st, x_img + (size_t)i * kXChunkBytes, kXChunkBytes, &rg.full[rg.p_stage], rg.pol_x);
        if (++rg.p_stage == rg.ns) { rg.p_stage = 0; rg.p_phase ^= 1; }
      }
      rg.pre = 0;
      if (next != nullptr && next->nrows != 0) prefetch_weights(rg, *next, w_img, ctrl);
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int c = (warp >> 2) - 1;        // this warpgroup's consumer
    if (c < ep.ncons) {
      int w_row0 = 0, acol = ep.col0;
      for (int i = 0; i < c; ++i) { w_row0 += 2 * ep.n[i]; acol += ep.n[i]; }
      if (ep.n[c] == 32) event_wg<64>(rg, chunks, w_row0, s_acc, acol, ctrl);
      else if (!kAllWidths || ep.n[c] == 16) event_wg<32>(rg, chunks, w_row0, s_acc, acol, ctrl);
      else if (ep.n[c] == 24) event_wg<48>(rg, chunks, w_row0, s_acc, acol, ctrl);
      else event_wg<16>(rg, chunks, w_row0, s_acc, acol, ctrl);
    } else {                              // no rows for this warpgroup: it still releases every stage it was counted for
      for (int i = 0; i < chunks; ++i) {
        mbar_wait(&rg.full[rg.c_stage], rg.c_phase, ctrl, 201);
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&rg.empty[rg.c_stage]);
        if (++rg.c_stage == rg.ns) { rg.c_stage = 0; rg.c_phase ^= 1; }
      }
    }
  }
  __syncthreads();
}

// keep bits (bit i = element idx0+i is kept) of 8 consecutive dropout elements, Philox4x32-10 one block per 4
__device__ __forceinline__ uint32_t philox_keep8(uint64_t seed, uint32_t site, uint64_t idx0, float pdrop) {
  uint32_t bits = 0;
  uint64_t blk_cur = ~0ull;
  uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint64_t idx = idx0 + i, blk = idx >> 2;
    if (blk != blk_cur) {
      philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), site, 0x7ac07201u, (uint32_t)seed, (uint32_t)(seed >> 32), o);
      blk_cur = blk;
    }
    const float u = (float)(o[idx & 3] >> 8) * (1.0f / 16777216.0f);
    bits |= (u >= pdrop ? 1u : 0u) << i;
  }
  return bits;
}

// accumulator columns [base + col, base + col + 8) of batch row `row`, then zero them (they are consumed)
__device__ __forceinline__ void acc_take8(float* s_acc, int row, int base, int col, float* s) {
  float* a = s_acc + row * kAccPitch + base + col;
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = a[i]; a[i] = 0.f; }
}

// training stash (decoder.h DecoderStash): gate activations, cell state and (post-dropout) hidden state of
// units [unit0, unit0 + 2) of batch row b at step t, fp32, PyTorch gate order
__device__ __forceinline__ void stash_lstm(float* gates, float* cs, float* hs, int t, int Btot, int b, int unit0,
                                           const float (&sg)[4][2], const float (&c)[2], const float (&h)[2]) {
  float* gp = gates + ((long)t * Btot + b) * (4 * kARnn) + unit0;
#pragma unroll
  for (int g = 0; g < 4; ++g) *reinterpret_cast<float2*>(gp + g * kARnn) = make_float2(sg[g][0], sg[g][1]);
  const long o = ((long)(t + 1) * Btot + b) * kARnn + unit0;
  *reinterpret_cast<float2*>(cs + o) = make_float2(c[0], c[1]);
  *reinterpret_cast<float2*>(hs + o) = make_float2(h[0], h[1]);
}

struct KParams {
  const CtaPlan* plans;
  const uint8_t* wimg;
  const float* bias_a; const float* bias_d; const float* bias_p;
  const uint8_t* weff_img; const float* w_v;
  // tensors
  const float* memory; const float* pm; const int32_t* mem_len;
  const uint8_t* prenet_keep; const uint8_t* att_keep; const uint8_t* dec_keep;
  // activation images (workspace)
  uint8_t* x2_img; uint8_t* ah_img; uint8_t* ctx_img; uint8_t* dh_img; uint8_t* x1_img;
  const uint8_t* teacher_x2_img;   // (cap, 4 chunks) or null
  float* q;                         // (64, 128) fp32
  float* mel; float* gate; float* align; int32_t* mel_lengths; int32_t* n_steps;
  DecoderCtrl* ctrl;
  int B, T, cap, infer, training;
  int nstages;                      // operand ring stages (4, or 3 when T_enc > 896)
  int t4max;                        // longest T_enc that runs with 4 stages (0: every T_enc runs with 3)
  int b0, Btot;                     // this launch handles batch rows [b0, b0 + B) of Btot (dropout mask / Philox indexing)
  float gate_threshold, score_mask_value, p_att, p_dec;
  uint64_t seed;
  DecoderStash st;                  // training stash for the backward pass (st.ga == nullptr: none)
  int t_begin, t_end;               // this launch runs steps [t_begin, t_end); the whole loop: 0, cap
  // resumable stream (t2_decoder_stream_run; rs_acc == nullptr: none).  The prologue restores and the epilogue saves the
  // on-chip state that lives past a step boundary; the activation images, q and the processed memory stay in place.
  float* rs_acc;                    // (kG, kRows x kAccPitch) accumulator tiles: next-step partial products
  float* rs_cell;                   // (kG, 4 column groups, kRows) float4 {c_att[0], c_att[1], c_dec[0], c_dec[1]}
  float* rs_att;                    // (kG, 2, padded TP) previous | cumulative attention weights
  int32_t* rs_done;                 // (kRows) stop latch
  int32_t* rs_status;               // out: [steps run, stopped]
};

// encoder-memory rows of a T_enc-long row that the attention phase stages in an idle ring of `nstages` stages; the rest
// is read from L2.  The same on the host and the device: the context of a row sums its positions in the grouping a
// launch sized for that row's own length stages (see the context below).
__host__ __device__ constexpr int staged_rows(int T, int nstages) {
  return T < (nstages * kStageBytes - 2 * kAttPlane - kPaBytes) / (kEnc / 2 * 4)
             ? T : (nstages * kStageBytes - 2 * kAttPlane - kPaBytes) / (kEnc / 2 * 4);
}

__device__ __forceinline__ void store_split2(uint8_t* img, int row, int k, float v0, float v1) {
  // two adjacent K elements (k even) of an activation image: 4-byte stores into the hi and lo planes
  const int chunk = k >> 6, kc = k & 63;
  __half h0, l0, h1, l1;
  split_fp16(v0, h0, l0);
  split_fp16(v1, h1, l1);
  __half* hi = reinterpret_cast<__half*>(img + (size_t)chunk * kXChunkBytes);
  __half* lo = hi + kRows * kChunkK;
  const uint32_t e = img_elem_offset(row, kc);
  *reinterpret_cast<__half2*>(hi + e) = __halves2half2(h0, h1);
  *reinterpret_cast<__half2*>(lo + e) = __halves2half2(l0, l1);
}

// ---------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1) decoder_persistent_kernel(const KParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x;
  const int T = p.T, TP = T + kLocK - 1;
  const int ntiles = (T + 127) >> 7;

  // ---- shared memory carve-up ----
  Carve sc(smem_raw, 1);
  PersistentSmem sm;
  persistent_smem_layout(sc, T, p.nstages, &sm);
  Ring rg;
  rg.ns = (uint32_t)p.nstages;
  rg.stage0 = sm.stage0;
  uint8_t* s_weff = sm.weff;
  float* s_acc = sm.acc;
  rg.full = sm.bars; rg.empty = sm.bars + kMaxStages;
  int* s_live = sm.live;
  int* s_flag = s_live + 1;
  float *s_bias_a = sm.bias_a, *s_bias_d = sm.bias_d, *s_v = sm.v, *s_q = sm.q;
  uint32_t* s_mask = sm.mask;
  float* s_bias_p = sm.bias_p;
  long long* s_prof = sm.prof;
  float *s_pad0 = sm.pad0, *s_pad1 = sm.pad1;
  float* s_e = sm.e;
  float* s_ep = sm.ep;     // one writer per (group, position), summed in a fixed order -> bit-reproducible

  rg.p_stage = rg.p_phase = rg.c_stage = rg.c_phase = 0;
  rg.pre = 0;

  if (tid == 0) {
    for (int s = 0; s < p.nstages; ++s) { ptx::mbar_init(&rg.full[s], 1); ptx::mbar_init(&rg.empty[s], kMmaWgs); }
    ptx::fence_barrier_init();
  }
  const bool resume = p.rs_acc != nullptr;       // a stream's chunk: its state was zeroed by begin or saved by the last chunk
  const int tpp = (TP + 3) & ~3;
  for (int i = tid; i < kRows * kAccPitch; i += kThreads)                  // every MMA accumulates
    s_acc[i] = resume ? p.rs_acc[(size_t)cta * kRows * kAccPitch + i] : 0.f;
  for (int i = tid; i < 32; i += kThreads) { s_bias_a[i] = p.bias_a[cta * 32 + i]; s_bias_d[i] = p.bias_d[cta * 32 + i]; }
  for (int i = tid; i < kWeffBytes / 16; i += kThreads)
    reinterpret_cast<uint4*>(s_weff)[i] = reinterpret_cast<const uint4*>(p.weff_img)[i];
  // The weight image (73.5 MiB, all of it streamed every step) is larger than the 50 MB L2, so its lines are marked to go
  // first; the activation chunks that every CTA reads keep evict_last.  Keeping half of the weight lines with evict_last
  // priority instead made the decoder step ~9 µs slower on H100 (DESIGN §6.1).
  rg.pol_w = ptx::policy_evict_first();
  rg.pol_x = ptx::policy_evict_last();
  for (int i = tid; i < kAtt; i += kThreads) s_v[i] = p.w_v[i];
  if (tid < 8) s_bias_p[tid] = (cta >= kPCta0 && cta < kPCta0 + kPCtas) ? p.bias_p[(cta - kPCta0) * 8 + tid] : 0.f;
  for (int i = tid; i < TP; i += kThreads) {                                        // model.py:274-277
    s_pad0[i] = resume ? p.rs_att[((size_t)cta * 2 + 0) * tpp + i] : 0.f;
    s_pad1[i] = resume ? p.rs_att[((size_t)cta * 2 + 1) * tpp + i] : 0.f;
  }
  const CtaPlan& plan = p.plans[cta];
  DecoderCtrl* ctrl = p.ctrl;
  const bool has_p = cta >= kPCta0 && cta < kPCta0 + kPCtas;
  const bool gate_cta = has_p && (cta - kPCta0) * 8 <= kMel && (cta - kPCta0) * 8 + 8 > kMel;   // owns the gate column
  if (resume && gate_cta && tid < p.B) ctrl->done[tid] = p.rs_done[tid];
  ptx::fence_proxy_async();       // s_weff is read by wgmma (async proxy)
  __syncthreads();

  unsigned int bar_target = 0;
  // epilogue role of this thread: quad = warp % 4, column group cg = warp / 4.  Quadrants 0/1 own batch rows
  // 0-63 (row = accumulator row); the threads of quadrants 2/3 (is_lo) take side jobs (dropout bits).
  const int quad = warp & 3, cg = warp >> 2;
  const int row = (quad & 1) * 32 + lane;               // batch row of this lane
  const bool is_lo = quad >= 2;
  const bool erow = !is_lo && row < p.B;
  float c_att[2] = {0.f, 0.f}, c_dec[2] = {0.f, 0.f};  // cell states of units 8*cta + 2*cg + {0,1}
  float4* rs_cell = resume ? reinterpret_cast<float4*>(p.rs_cell) + ((size_t)cta * 4 + cg) * kRows + row : nullptr;
  if (resume && !is_lo) {
    const float4 c = *rs_cell;
    c_att[0] = c.x; c_att[1] = c.y; c_dec[0] = c.z; c_dec[1] = c.w;
  }
  const bool has_q = cta >= kQCta0 && cta < kQCta0 + kQCtas;
  const bool has_x2 = cta >= kX2Cta0 && cta < kX2Cta0 + kX2Ctas;
  const int halfk = (kLocK - 1) / 2;
  // phase profile (cycles, accumulated over steps) on three sample CTAs; see t2_decoder_profile()
  const int prof_slot = cta == 0 ? 0 : (cta == 60 ? 1 : (cta == 100 ? 2 : -1));
  long long prof_last = clock64();
  if (tid < 24) s_prof[tid] = 0;
#define T2_PROF(ph)                                                        \
  do {                                                                     \
    if (prof_slot >= 0 && tid == 0) {                                      \
      const long long now_ = clock64();                                    \
      s_prof[ph] += now_ - prof_last;   /* shared memory: a global read-modify-write here stalls the producer thread */ \
      prof_last = now_;                                                    \
    }                                                                      \
  } while (0)
  // LSTM epilogue shared by both cells: take the 8 gate columns (2 units x i,f,g,o) of this lane's batch row
#define T2_TAKE_GATES(colbase, g)                          \
  do {                                                     \
    if (!is_lo) acc_take8(s_acc, row, (colbase), cg * 8, g); \
  } while (0)

  // epilogue of E4 on the prenet-2 CTAs: x2 = relu(W_2 x1) * mask * 2 -> x2 image            model.py:97-100
  auto x2_epilogue = [&]() {
    float g[8];
    if (cg == 0 && !is_lo) acc_take8(s_acc, row, kColS, 0, g);
    if (cg == 0 && erow) {
      const int col0 = (cta - kX2Cta0) * 8;
      float r[8];
      const uint32_t bits = s_mask[row];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        r[j] = ((bits >> j) & 1u) ? fmaxf(g[j], 0.f) * 2.f : 0.f;
#pragma unroll
      for (int j = 0; j < 8; j += 2) store_split2(p.x2_img, row, col0 + j, r[j], r[j + 1]);
    }
  };

  // the hand-over counters and the grid barrier count from zero in every launch: their targets are relative to t_begin,
  // while dropout keys, output indices and the stop test use the absolute step t
  int t = p.t_begin;
  for (; t < p.t_end; ++t) {
    // ======== E0: x2_t -> attention LSTM gates, epilogue -> ah_t ==================== model.py:352-356
    {
      const uint8_t* x2 = p.infer ? p.x2_img : p.teacher_x2_img + (size_t)t * 4 * kXChunkBytes;
      run_event(rg, plan.ev[0], x2, p.wimg, 4, s_acc, ctrl, &plan.ev[1]);
      T2_PROF(0);
      float g[8];
      T2_TAKE_GATES(kColA, g);
      if (erow) {
        float hv[2], sg[4][2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float* b = s_bias_a + (cg * 2 + u) * 4;
          const float gi = sigmoid_fast(g[u * 4 + 0] + b[0]);
          const float gf = sigmoid_fast(g[u * 4 + 1] + b[1]);
          const float gg = tanh_fast(g[u * 4 + 2] + b[2]);
          const float go = sigmoid_fast(g[u * 4 + 3] + b[3]);
          c_att[u] = gf * c_att[u] + gi * gg;
          float h = go * tanh_fast(c_att[u]);
          if (p.training) {
            const int unit = cta * 8 + cg * 2 + u;
            const long idx = (long)(p.b0 + row) * kARnn + unit;
            const bool keep = p.att_keep ? p.att_keep[(long)t * p.Btot * kARnn + idx] != 0
                                         : philox_keep(p.seed, t * 4 + 2, idx, p.p_att);
            h = keep ? h * (1.f / (1.f - p.p_att)) : 0.f;
          }
          hv[u] = h;
          sg[0][u] = gi; sg[1][u] = gf; sg[2][u] = gg; sg[3][u] = go;
        }
        store_split2(p.ah_img, row, cta * 8 + cg * 2, hv[0], hv[1]);
        if (p.st.ga) stash_lstm(p.st.ga, p.st.ca, p.st.ha, t, p.Btot, p.b0 + row, cta * 8 + cg * 2, sg, c_att, hv);
      }
      T2_PROF(1);
      signal_counter(&ctrl->ah_count[cta >> 3], 1u);                        // this CTA's 8 columns of ah_t are written
      T2_PROF(2);
    }
    // ======== E1: ah_t -> dec gates (part), next att gates (part), query ===== model.py:57, 366-369
    {
      // while the producer / MMA threads stream this event, the otherwise idle lo-row lanes of column group 0
      // (warps 2, 3) draw the prenet dropout bits this CTA needs at the END of this step (x1 columns on the projection CTAs, x2 columns on the prenet-2 CTAs)
      if (p.infer && is_lo && cg == 0 && row < p.B && t + 1 < p.cap && (has_p || has_x2)) {
        uint32_t bits = 0;
        if (has_x2) {
          const int col0 = (cta - kX2Cta0) * 8;
          if (p.prenet_keep) {
            const uint8_t* kp = p.prenet_keep + ((long)(t + 1) * 2 + 1) * p.Btot * kPre + (long)(p.b0 + row) * kPre + col0;
            for (int j = 0; j < 8; ++j) bits |= (kp[j] != 0 ? 1u : 0u) << j;
          } else {
            bits = philox_keep8(p.seed, (t + 1) * 4 + 1, (uint64_t)(p.b0 + row) * kPre + col0, 0.5f);
          }
        } else {
          const int pc0 = (cta - kPCta0) * 8;
          for (int j = 0; j < 8; ++j) {
            const int col = pc0 + j - (kMel + 1);
            if (col < 0 || col >= kPre) continue;
            const long idx = (long)(p.b0 + row) * kPre + col;
            const bool keep = p.prenet_keep ? p.prenet_keep[((long)(t + 1) * 2 + 0) * p.Btot * kPre + idx] != 0
                                            : philox_keep(p.seed, (t + 1) * 4 + 0, idx, 0.5f);
            bits |= (keep ? 1u : 0u) << j;
          }
        }
        s_mask[row] = bits;
      }
      run_event(rg, plan.ev[1], p.ah_img, p.wimg, 16, s_acc, ctrl, nullptr,    // the attention phase reuses the ring as scratch
                ctrl->ah_count, 8u * (unsigned int)(t + 1 - p.t_begin));
      if (has_q && cg == 0 && !is_lo) {
        float g[8];
        acc_take8(s_acc, row, kColS, 0, g);
        if (erow) {
#pragma unroll
          for (int j = 0; j < 8; ++j) p.q[row * kAtt + (cta - kQCta0) * 8 + j] = g[j];
        }
      }
      T2_PROF(3);
    }
    // ======== attention for batch row (cta mod 64) ============================ model.py:43-86, 358-365
    // CTAs b and b+64 both evaluate row b's energies / softmax (no exchange needed, bit-identical); each
    // produces one half of the context columns, the first writes the alignment row.  Everything that only
    // needs THIS CTA's state (im2col of its attention weights, the pa GEMM, staging encoder memory rows)
    // runs between the arrival at barrier B2 and the wait for it.
    const bool att_cta = (cta & 63) < p.B;
    const int att_b = cta & 63, ahalf = cta >> 6;
    uint8_t* aimg = rg.stage0;
    // the idle operand ring during the attention phase: [im2col image: hi plane | lo plane][pa tile][encoder-memory rows
    // of this CTA]
    const int att_rounds = (T + kAttRound - 1) / kAttRound;
    const int img_bytes = 2 * kAttPlane;
    float* s_pa = reinterpret_cast<float*>(aimg + img_bytes);                       // [128 dims][kPaPitch] fp32
    const int smem_rows = staged_rows(T, p.nstages);                        // memory rows staged in the ring
    // pa^T = Weff . A^T on the tensor cores (fused model.py:23-25), i.e. the fused filter bank is the M = 128 operand
    // (attention dim d; warpgroups 0 / 1 take dims 0-63 / 64-127) and kAttRound positions are the N dimension.  The
    // tile goes to shared memory, where every warp then owns a slice of POSITIONS of all 128 dims, so the tanh of a
    // row spread evenly over the four SM sub-partitions for any T_enc, the processed-memory reads are coalesced
    // (lanes = consecutive dims) and can be issued before the q barrier.
    auto att_im2col_mma_tr = [&](int r0) {
      const int jbase = r0 * kAttRound, cnt = min(T - jbase, kAttRound);
      for (int item = tid; item < kAttRound * 8; item += kThreads) {
        const int jj = item >> 3, g8 = item & 7, j = jbase + jj;
        __align__(16) __half hh[8];
        __align__(16) __half ll[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int kk = g8 * 8 + e;
          float v = 0.f;
          if (jj < cnt && kk < 2 * kLocK) v = kk < kLocK ? s_pad0[j + kk] : s_pad1[j + kk - kLocK];
          split_fp16(v, hh[e], ll[e]);
        }
        uint8_t* dst = aimg + (jj >> 3) * 1024 + (jj & 7) * 128 + ((g8 ^ (jj & 7)) * 16);
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hh);
        *reinterpret_cast<uint4*>(dst + kAttPlane) = *reinterpret_cast<const uint4*>(ll);
      }
      ptx::fence_proxy_async();
      __syncthreads();
      if (warp < 8) {
        const int wg = warp >> 2, wt = tid & 127;
        const uint32_t ws = ptx::smem_u32(s_weff) + (uint32_t)wg * (64 * 128), ps = ptx::smem_u32(aimg);
        float d[kAttRound / 2];
#pragma unroll
        for (int i = 0; i < kAttRound / 2; ++i) d[i] = 0.f;
        ptx::wg_fence_regs<kAttRound / 2>(d);
        ptx::wg_fence();
#pragma unroll
        for (int kk = 0; kk < kChunkK / 16; ++kk) {
          const uint64_t w_hi = ptx::make_sw128_desc(ws + kk * 32);
          const uint64_t w_lo = ptx::make_sw128_desc(ws + kAtt * 128 + kk * 32);
          const uint64_t p_hi = ptx::make_sw128_desc(ps + kk * 32);
          const uint64_t p_lo = ptx::make_sw128_desc(ps + kAttPlane + kk * 32);
          ptx::wgmma_f16<kAttRound>(d, w_hi, p_hi);
          ptx::wgmma_f16<kAttRound>(d, w_lo, p_hi);
          ptx::wgmma_f16<kAttRound>(d, w_hi, p_lo);
        }
        ptx::wg_commit();
        ptx::wg_wait<0>();
        ptx::wg_fence_regs<kAttRound / 2>(d);
#pragma unroll
        for (int i = 0; i < kAttRound / 2; i += 2)
          *reinterpret_cast<float2*>(s_pa + (wg * 64 + ptx::wg_frag_row(i, wt)) * kPaPitch + ptx::wg_frag_col(i, wt)) =
              make_float2(d[i], d[i + 1]);
      }
      __syncthreads();
    };
    auto stage_memory_rows = [&](int j0, int j1) {     // cp.async this CTA's half of memory rows [j0, j1) into the ring
      const uint32_t sbase = ptx::smem_u32(rg.stage0) + (uint32_t)(img_bytes + kPaBytes);
      const float* msrc = p.memory + (long)att_b * T * kEnc + ahalf * (kEnc / 2);
      for (int i = j0 * 64 + tid; i < j1 * 64; i += kThreads) {
        const int j = i >> 6, c4 = i & 63;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sbase + (uint32_t)i * 16u),
                     "l"(msrc + (long)j * kEnc + c4 * 4)
                     : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    grid_arrive(ctrl, bar_target);                                             // B2 (arrive): q written
    const int adim = quad * 32 + lane;     // this thread's attention dim
    float pm_next[8];                      // processed-memory values of the thread's next chunk of 8 positions (software pipeline)
    auto load_pm = [&](const float* pmr, int j0, int cnt) {
#pragma unroll
      for (int e = 0; e < 8; ++e) pm_next[e] = (j0 + e < cnt) ? __ldg(pmr + (long)(j0 + e) * kAtt) : 0.f;
    };
    if (att_cta) {
      att_im2col_mma_tr(0);
      stage_memory_rows(0, smem_rows);     // everything the context needs is in flight before the q barrier
      load_pm(p.pm + (long)att_b * T * kAtt + adim, cg * 8, min(T, kAttRound));
    }
    T2_PROF(15);
    grid_wait(ctrl, bar_target);                                               // B2 (wait): q complete
    T2_PROF(4);
    if (att_cta) {
      const int b = att_b;
      for (int i = tid; i < kAtt; i += kThreads) s_q[i] = __ldcg(&p.q[b * kAtt + i]);
      __syncthreads();
      {
        const int eN = ntiles * 128;
        const float qd = s_q[adim], vd = s_v[adim];
        const int nrounds = att_rounds;
        for (int r0 = 0; r0 < nrounds; ++r0) {
          const int jbase = r0 * kAttRound, cnt = min(T - jbase, kAttRound), nch = (cnt + 7) >> 3;
          if (r0 > 0) att_im2col_mma_tr(r0);
          T2_PROF(16);
          // energies e_j = sum_d v_d tanh(q_d + pa_dj + pm_jd): this thread adds dim d = adim for the 8 positions of
          // each of its chunks, then the 32 dims of the warp are summed with a transpose-reduce (9 shuffles per 8
          // positions, fixed order); the four 32-dim groups of a position are added in a fixed order at the softmax
          const float* pmr = p.pm + ((long)b * T + jbase) * kAtt + adim;
          if (r0 > 0) load_pm(pmr, cg * 8, cnt);
#pragma unroll 1
          for (int c = cg; c < nch; c += 4) {
            const int j0 = c * 8;
            float pm8[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) pm8[e] = pm_next[e];
            if (c + 4 < nch) load_pm(pmr, j0 + 32, cnt);           // next chunk's loads fly during this chunk's tanh
            float g[8], sv[8];
            {
              const float4 g0 = *reinterpret_cast<const float4*>(s_pa + adim * kPaPitch + j0);
              const float4 g1 = *reinterpret_cast<const float4*>(s_pa + adim * kPaPitch + j0 + 4);
              g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) sv[e] = vd * tanh_fast(qd + g[e] + pm8[e]);
            float r4[4], r2[2], r1;
            {
              const bool up = (lane & 16) != 0;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float send = up ? sv[e] : sv[e + 4], keep = up ? sv[e + 4] : sv[e];
                r4[e] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
            }
            {
              const bool up = (lane & 8) != 0;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float send = up ? r4[e] : r4[e + 2], keep = up ? r4[e + 2] : r4[e];
                r2[e] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
            }
            {
              const bool up = (lane & 4) != 0;
              const float send = up ? r2[0] : r2[1], keep = up ? r2[1] : r2[0];
              r1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
            r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
            const int jj = j0 + ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
            if ((lane & 3) == 0 && jj < cnt) s_ep[quad * eN + jbase + jj] = r1;
          }
          __syncthreads();
          T2_PROF(17);
        }
      }
      // mask + softmax (model.py:79-82): every warp reduces all T energies itself (shuffles only, no
      // cross-warp exchange), then the threads split the normalised write-out
      const int len = p.mem_len ? min(p.mem_len[b], T) : T;
      const int eN = ntiles * 128;
      // masked energies once (the four 32-dim partial sums added in a fixed order), in place in the first partial-sum plane
      for (int j = tid; j < T; j += kThreads)
        s_ep[j] = (j < len) ? (s_ep[j] + s_ep[eN + j]) + (s_ep[2 * eN + j] + s_ep[3 * eN + j]) : p.score_mask_value;
      __syncthreads();
      float mx = -INFINITY;
      for (int j = lane; j < T; j += 32) mx = fmaxf(mx, s_ep[j]);
      mx = warp_max_f(mx);
      float sum = 0.f;
      for (int j = lane; j < T; j += 32) sum += expf(s_ep[j] - mx);
      sum = warp_sum_f(sum);
      const float inv = 1.f / sum;
      for (int j = tid; j < T; j += kThreads) {
        const float a = expf(s_ep[j] - mx) * inv;
        s_e[j] = a;
        s_pad0[halfk + j] = a;                                                // becomes "previous"
        s_pad1[halfk + j] += a;                                               // model.py:365
        if (ahalf == 0) p.align[((long)b * p.cap + t) * T + j] = a;
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      T2_PROF(18);
      {                                                           // context = aw . memory  model.py:83-84
        // j-group jg sums positions jg, jg + 8, ... below `split`, then split + jg, split + jg + 8, ... below `clen`.
        // INFER: clen = len and split = the rows a launch sized for T_enc = len stages, so the grouping is a function of
        // the row's own length, not of the launch's T_enc, and a row of a ragged batch gets the bits it gets alone
        // (positions >= len have weight 0 and are skipped).  Without lengths, len = T_enc and split = smem_rows.
        // TEACHER keeps the launch's grouping over all T_enc positions.
        const int c4 = tid & 63, jg = tid >> 6;                   // 64 float4 = this CTA's 256 columns; 8 j-groups
        const float4* ms = reinterpret_cast<const float4*>(rg.stage0 + img_bytes + kPaBytes);
        const float* mp = p.memory + (long)b * T * kEnc + ahalf * (kEnc / 2) + c4 * 4;
        const int clen = p.infer ? len : T;
        const int split = p.infer ? staged_rows(len, len <= p.t4max ? 4 : 3) : smem_rows;   // >= smem_rows if clen > smem_rows
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int j = jg;
#pragma unroll 4
        for (; j < min(split, smem_rows); j += 8) {
          const float4 m = ms[j * 64 + c4];
          const float a = s_e[j];
          acc.x = fmaf(a, m.x, acc.x); acc.y = fmaf(a, m.y, acc.y); acc.z = fmaf(a, m.z, acc.z); acc.w = fmaf(a, m.w, acc.w);
        }
        for (; j < split; j += 8) {                               // staged for a launch of this length, not for this one
          const float4 m = __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc));
          const float a = s_e[j];
          acc.x = fmaf(a, m.x, acc.x); acc.y = fmaf(a, m.y, acc.y); acc.z = fmaf(a, m.z, acc.z); acc.w = fmaf(a, m.w, acc.w);
        }
        for (j = split + jg; j < clen; j += 8) {                  // rows that did not fit in the ring
          const float4 m = __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc));
          const float a = s_e[j];
          acc.x = fmaf(a, m.x, acc.x); acc.y = fmaf(a, m.y, acc.y); acc.z = fmaf(a, m.z, acc.z); acc.w = fmaf(a, m.w, acc.w);
        }
        __syncthreads();                                          // everyone is done reading the staged rows
        float* scr = reinterpret_cast<float*>(rg.stage0);         // [8][256] partial sums
        *reinterpret_cast<float4*>(scr + jg * (kEnc / 2) + c4 * 4) = acc;
        __syncthreads();
        if (tid < kEnc / 4) {
          const int col = tid * 2;
          float v0 = 0.f, v1 = 0.f;
#pragma unroll
          for (int g = 0; g < 8; ++g) { v0 += scr[g * (kEnc / 2) + col]; v1 += scr[g * (kEnc / 2) + col + 1]; }
          store_split2(p.ctx_img, b, ahalf * (kEnc / 2) + col, v0, v1);
          if (p.st.ga)
            *reinterpret_cast<float2*>(p.st.ctx + ((long)(t + 1) * p.Btot + p.b0 + b) * kEnc + ahalf * (kEnc / 2) + col) =
                make_float2(v0, v1);
        }
      }
      T2_PROF(19);
    }
    T2_PROF(5);
    grid_barrier(ctrl, bar_target);                                                             // B3: ctx_t complete
    T2_PROF(6);
    // ======== E2: ctx_t -> dec gates (rest), next att gates, projection (part); epilogue -> dh_t
    {
      run_event(rg, plan.ev[2], p.ctx_img, p.wimg, 8, s_acc, ctrl, &plan.ev[3]);
      T2_PROF(7);
      float g[8];
      T2_TAKE_GATES(kColD, g);
      if (erow) {
        float hv[2], sg[4][2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float* b = s_bias_d + (cg * 2 + u) * 4;
          const float gi = sigmoid_fast(g[u * 4 + 0] + b[0]);
          const float gf = sigmoid_fast(g[u * 4 + 1] + b[1]);
          const float gg = tanh_fast(g[u * 4 + 2] + b[2]);
          const float go = sigmoid_fast(g[u * 4 + 3] + b[3]);
          c_dec[u] = gf * c_dec[u] + gi * gg;
          float h = go * tanh_fast(c_dec[u]);
          if (p.training) {
            const int unit = cta * 8 + cg * 2 + u;
            const long idx = (long)(p.b0 + row) * kDRnn + unit;
            const bool keep = p.dec_keep ? p.dec_keep[(long)t * p.Btot * kDRnn + idx] != 0
                                         : philox_keep(p.seed, t * 4 + 3, idx, p.p_dec);
            h = keep ? h * (1.f / (1.f - p.p_dec)) : 0.f;
          }
          hv[u] = h;
          sg[0][u] = gi; sg[1][u] = gf; sg[2][u] = gg; sg[3][u] = go;
        }
        store_split2(p.dh_img, row, cta * 8 + cg * 2, hv[0], hv[1]);
        if (p.st.ga) stash_lstm(p.st.gd, p.st.cd, p.st.hd, t, p.Btot, p.b0 + row, cta * 8 + cg * 2, sg, c_dec, hv);
      }
      T2_PROF(8);
      signal_counter(&ctrl->dh_count[cta >> 3], 1u);                        // this CTA's 8 columns of dh_t are written
      T2_PROF(9);
    }
    // ======== E3: dh_t -> projection (rest), next dec gates (part); epilogue -> mel, gate, x1
    {
      run_event(rg, plan.ev[3], p.dh_img, p.wimg, 16, s_acc, ctrl,
                (!p.infer && t + 1 < p.cap) ? &plan.ev[0] : nullptr,    // INFER: the loop may end after this step
                ctrl->dh_count, 8u * (unsigned int)(t + 1 - p.t_begin));
      T2_PROF(10);
      if (tid == 0) *s_live = 0;
      float g[8];
      if (has_p && cg == 0 && !is_lo) acc_take8(s_acc, row, kColS, 0, g);
      __syncthreads();                                                         // s_live is reset before anyone counts
      if (has_p && cg == 0 && erow) {
        const int pc0 = (cta - kPCta0) * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int pc = pc0 + j;
          const float v = g[j] + s_bias_p[j];
          if (pc < kMel) {
            p.mel[((long)row * p.cap + t) * kMel + pc] = v;                    // model.py:375-376
          } else if (pc == kMel) {
            p.gate[(long)row * p.cap + t] = v;                                 // model.py:378
            if (p.infer) {
              int done = ctrl->done[row];
              if (!done && sigmoid_exact(v) > p.gate_threshold) {             // model.py:443
                done = 1; ctrl->done[row] = 1; p.mel_lengths[row] = t + 1;
              }
              if (!done) atomicAdd(s_live, 1);
            }
          } else if (pc < kMel + 1 + kPre) {                                   // first prenet layer of step t+1
            const int col = pc - (kMel + 1);
            float r = fmaxf(v, 0.f);
            if (p.infer && t + 1 < p.cap) r = ((s_mask[row] >> j) & 1u) ? r * 2.f : 0.f;
            if (p.infer) {
              __half h, l;
              split_fp16(r, h, l);
              __half* hi = reinterpret_cast<__half*>(p.x1_img + (size_t)(col >> 6) * kXChunkBytes);
              __half* lo = hi + kRows * kChunkK;
              const uint32_t e = img_elem_offset(row, col & 63);
              hi[e] = h; lo[e] = l;
            }
          }
        }
      }
      __syncthreads();
      if (gate_cta && tid == 0) atomicMax(p.n_steps, t + 1);
      T2_PROF(11);
      if (!p.infer) continue;                                                  // teacher forcing: x2 is precomputed
      // x1 has 43 producers (the projection CTAs) and 32 consumers (the prenet-2 CTAs), x2 has those 32 producers and
      // everybody as consumer: two producer-scoped arrival counters instead of two 128-way barriers -- nobody but
      // the 32 prenet-2 CTAs waits for x1.  The stop decision rides on the counters (bits 24+): the gate CTA adds
      // kStopFlag to its x1 arrival when every row has fired, the prenet-2 CTAs pass it on with their x2 arrival.
      bool stop = t + 1 == p.cap;
      if (has_p) signal_counter(&ctrl->x1_count, 1u + ((gate_cta && *s_live == 0) ? kStopFlag : 0u));
      if (has_x2) {
        stop |= wait_counter(&ctrl->x1_count, (unsigned int)(kPCtas * (t + 1 - p.t_begin)), s_flag, ctrl, 102);
        if (!stop) {
          run_event(rg, plan.ev[4], p.x1_img, p.wimg, 4, s_acc, ctrl, nullptr);    // E4: x1 -> x2_(t+1)  model.py:97-100
          x2_epilogue();
        }
        signal_counter(&ctrl->x2_count, 1u + (stop ? kStopFlag : 0u));
      }
      T2_PROF(12);
      stop |= wait_counter(&ctrl->x2_count, (unsigned int)(kX2Ctas * (t + 1 - p.t_begin)), s_flag, ctrl, 103);
      T2_PROF(14);
      if (stop) { ++t; break; }
    }
  }
  if (prof_slot >= 0 && tid == 0)
    for (int i = 0; i < 24; ++i) ctrl->prof[prof_slot][i] = s_prof[i];
  if (resume) {    // every step ended with a wait that closes with __syncthreads: the shared-memory state is complete
    for (int i = tid; i < kRows * kAccPitch; i += kThreads) p.rs_acc[(size_t)cta * kRows * kAccPitch + i] = s_acc[i];
    for (int i = tid; i < TP; i += kThreads) {
      p.rs_att[((size_t)cta * 2 + 0) * tpp + i] = s_pad0[i];
      p.rs_att[((size_t)cta * 2 + 1) * tpp + i] = s_pad1[i];
    }
    if (!is_lo) *rs_cell = make_float4(c_att[0], c_att[1], c_dec[0], c_dec[1]);
    if (gate_cta && tid < p.B) p.rs_done[tid] = ctrl->done[tid];
  }
  // rows that never fired: length = number of steps run (model.py:445-447)
  if (cta == 0) {
    __syncthreads();
    const int ns = p.infer ? t : p.cap;
    // a stream's chunk that reached t_end with rows still live and steps left has not ended the loop
    bool ended = true;
    if (resume) ended = t >= p.cap || __syncthreads_count(tid < p.B && !__ldcg(&ctrl->done[tid])) == 0;
    if (ended) {
      for (int b = tid; b < p.B; b += kThreads)
        if (!p.infer || !__ldcg(&ctrl->done[b])) p.mel_lengths[b] = ns;
      if (tid == 0) atomicMax(p.n_steps, ns);
    }
    if (resume && tid == 0) { p.rs_status[0] = t; p.rs_status[1] = ended ? 1 : 0; }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
constexpr size_t kSmemReserve = 1024;    // headroom past the last region
static size_t persistent_smem_bytes(int T, int nstages) {
  Carve c(nullptr, 1);
  PersistentSmem s;
  persistent_smem_layout(c, T, nstages, &s);
  return c.bytes() + kSmemReserve;
}
constexpr size_t kSmemLimit = 227 * 1024;
// 4 ring stages when they fit beside the T_enc-dependent attention state (T_enc <= 896 on sm_90's 227 KiB), else 3
// (T_enc <= 2274; longer memories are refused, see persistent_supported).  The idle ring stages encoder-memory rows
// 0-93 at 4 stages and 0-57 at 3 for the attention context; later rows are read from L2.
static int persistent_stages(int T) {
  int want = 4;
  const char* e = getenv("T2_STAGES");
  if (e && atoi(e) >= 3 && atoi(e) <= kMaxStages) want = atoi(e);
  while (want > 3 && persistent_smem_bytes(T, want) > kSmemLimit) --want;
  return want;
}

constexpr int kImageChunks = 4 + 16 + 8 + 16 + 4;          // K chunks of the x2, ah, ctx, dh and x1 images
constexpr size_t kImagesBytes = (size_t)kImageChunks * kXChunkBytes + (size_t)kRows * kAtt * 4;   // + q

// the persistent kernel's part of the decoder workspace: activation images x2 (4 chunks), ah (16), ctx (8), dh (16),
// x1 (4) and q (64 x 128 fp32); for teacher forcing the x2 images of every step (cap x 4 chunks)
void persistent_ws_layout(Carve& c, int cap, DecoderWs* w) {
  w->images = c.take<uint8_t>(kImagesBytes);
  w->teacher_img = c.take<uint8_t>((size_t)cap * 4 * kXChunkBytes, 1024);
}

bool persistent_supported(const T2Model* m, const T2DecoderArgs* a) {
  if (!m->pk) return false;
  if (m->sm_count < kG) return false;
  if (persistent_smem_bytes(a->T_enc, 3) > kSmemLimit) return false;
  return true;
}

int persistent_pack_create(T2Model* m, cudaStream_t s) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  if (!pk) { pk = new PersistentPack(); m->pk = pk; }
  const int kdc = kDRnn + kEnc;
  // ---- per-CTA plans (host).  Consumers of an event are a contiguous run of [A | D | S] ----
  std::vector<CtaPlan> plans(kG);
  size_t off = 0;
  for (int c = 0; c < kG; ++c) {
    const bool hq = c >= kQCta0 && c < kQCta0 + kQCtas, hx = c >= kX2Cta0 && c < kX2Cta0 + kX2Ctas,
               hp = c >= kPCta0 && c < kPCta0 + kPCtas;
    CtaPlan& pl = plans[c];
    memset(&pl, 0, sizeof(pl));
    auto set = [&](int ev, int chunks, int col0, std::initializer_list<int> ns) {
      EventPlan& e = pl.ev[ev];
      e.ncons = 0; e.nrows = 0; e.col0 = col0;
      for (int n : ns) { e.n[e.ncons++] = n; e.nrows += n; }
      e.w_bytes = (uint32_t)e.nrows * 256;
      e.w_off = (uint32_t)off;
      e.chunks = chunks;
      off += (size_t)chunks * e.w_bytes;
    };
    set(0, 4, kColA, {32});
    if (hq) set(1, 16, kColA, {32, 32, 16}); else set(1, 16, kColA, {32, 32});
    if (hp) set(2, 8, kColA, {32, 32, 16}); else set(2, 8, kColA, {32, 32});
    if (hp) set(3, 16, kColD, {32, 16}); else set(3, 16, kColD, {32});
    if (hx) set(4, 4, kColS, {16}); else { pl.ev[4].w_off = (uint32_t)off; }
    for (int ev = 0; ev < kNumEvents; ++ev)
      if (pl.ev[ev].nrows != 0 && !event_plan_fits(pl.ev[ev], false)) return fail(T2_ERR_INVALID, "event plan does not fit the MMA warpgroups");
  }
  if (off >= (size_t)4 << 30) return fail(T2_ERR_INVALID, "W image too large");
  const std::vector<BwdCta> bwd_plans[2] = {bwd_gemm_plans(0), bwd_gemm_plans(1)};
  if (!pk->wimg) {
    pk->wimg_bytes = off + 1024;
    T2_CUDA(cudaMalloc((void**)&pk->wimg, pk->wimg_bytes));
    T2_CUDA(cudaMalloc((void**)&pk->plans, sizeof(CtaPlan) * kG));
    T2_CUDA(cudaMalloc((void**)&pk->wp_all, (size_t)kPCols * kdc * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_p, (size_t)kPCols * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_a, (size_t)kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_d, (size_t)kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->rows, (size_t)4 * kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->weff, (size_t)kAtt * kChunkK * 4));
    T2_CUDA(cudaMalloc((void**)&pk->weff_img, (size_t)kWeffBytes));
    for (int which = 0; which < 2; ++which) T2_CUDA(cudaMalloc((void**)&pk->bwd_plans[which], sizeof(BwdCta) * bwd_plans[which].size()));
  }
  fuse_location_kernel<<<kAtt, kChunkK, 0, s>>>(m->w[W_ATT_LOC_DENSE], m->w[W_ATT_LOC_CONV], pk->weff);
  T2_LAUNCH_CHECK();
  pack_rows_image_kernel<<<1, 256, 0, s>>>(pk->weff, kAtt, kChunkK, pk->weff_img);
  T2_LAUNCH_CHECK();
  T2_CUDA(cudaMemcpyAsync(pk->plans, plans.data(), sizeof(CtaPlan) * kG, cudaMemcpyHostToDevice, s));
  for (int which = 0; which < 2; ++which)
    T2_CUDA(cudaMemcpyAsync(pk->bwd_plans[which], bwd_plans[which].data(), sizeof(BwdCta) * bwd_plans[which].size(),
                            cudaMemcpyHostToDevice, s));
  T2_CUDA(cudaStreamSynchronize(s));   // `plans` and `bwd_plans` are host temporaries
  // ---- W_P = [proj (80) ; gate (1) ; W1.Wproj (256) ; 0 (7)] and its bias ----
  T2_CUDA(cudaMemsetAsync(pk->wp_all, 0, (size_t)kPCols * kdc * 4, s));
  T2_CUDA(cudaMemsetAsync(pk->bias_p, 0, (size_t)kPCols * 4, s));
  T2_CUDA(cudaMemcpyAsync(pk->wp_all, m->projgate_w, (size_t)(kMel + 1) * kdc * 4, cudaMemcpyDeviceToDevice, s));
  T2_CUDA(cudaMemcpyAsync(pk->bias_p, m->projgate_b, (size_t)(kMel + 1) * 4, cudaMemcpyDeviceToDevice, s));
  fuse_prenet_proj_kernel<<<kPre, 256, 0, s>>>(m->w[W_PRENET0], m->w[W_PROJ_W], m->w[W_PROJ_B],
                                               pk->wp_all + (size_t)(kMel + 1) * kdc, pk->bias_p + kMel + 1);
  T2_LAUNCH_CHECK();
  pack_lstm_bias_kernel<<<(kG * 32 + 255) / 256, 256, 0, s>>>(m->arnn_b, pk->bias_a);
  T2_LAUNCH_CHECK();
  pack_lstm_bias_kernel<<<(kG * 32 + 255) / 256, 256, 0, s>>>(m->drnn_b, pk->bias_d);
  T2_LAUNCH_CHECK();
  // ---- row tables: [0] LSTM gate rows, [1] q rows, [2] P rows, [3] x2 rows (S consumers: 8 real + 8 zero) ----
  std::vector<int32_t> rows((size_t)4 * kG * 32, -1);
  for (int c = 0; c < kG; ++c) {
    for (int col = 0; col < 32; ++col) rows[(0 * kG + c) * 32 + col] = (col & 3) * 1024 + c * 8 + (col >> 2);
    if (c >= kQCta0 && c < kQCta0 + kQCtas) for (int j = 0; j < 8; ++j) rows[(1 * kG + c) * 32 + j] = (c - kQCta0) * 8 + j;
    if (c >= kPCta0 && c < kPCta0 + kPCtas) for (int j = 0; j < 8; ++j) rows[(2 * kG + c) * 32 + j] = (c - kPCta0) * 8 + j;
    if (c >= kX2Cta0 && c < kX2Cta0 + kX2Ctas) for (int j = 0; j < 8; ++j) rows[(3 * kG + c) * 32 + j] = (c - kX2Cta0) * 8 + j;
  }
  T2_CUDA(cudaMemcpyAsync(pk->rows, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
  T2_CUDA(cudaStreamSynchronize(s));
  const int32_t* r_lstm = pk->rows; const int32_t* r_q = pk->rows + kG * 32;
  const int32_t* r_p = pk->rows + 2 * kG * 32; const int32_t* r_x2 = pk->rows + 3 * kG * 32;
  auto pack = [&](const float* src, int ld, int kcol0, int chunks, const int32_t* rt, int ev, int cons) -> int {
    pack_consumer_kernel<<<dim3(chunks, kG), 256, 0, s>>>(src, ld, kcol0, rt, pk->plans, ev, cons, pk->wimg);
    T2_LAUNCH_CHECK();
    return T2_OK;
  };
  T2_TRY(pack(m->w[W_ARNN_WIH], kPre + kEnc, 0, 4, r_lstm, 0, 0));            // E0: att <- x2
  T2_TRY(pack(m->w[W_ARNN_WHH], kARnn, 0, 16, r_lstm, 1, 0));                 // E1: att' <- ah
  T2_TRY(pack(m->w[W_DRNN_WIH], kdc, 0, 16, r_lstm, 1, 1));                   //     dec <- ah
  T2_TRY(pack(m->w[W_ATT_QUERY], kARnn, 0, 16, r_q, 1, 2));                   //     q <- ah
  T2_TRY(pack(m->w[W_ARNN_WIH], kPre + kEnc, kPre, 8, r_lstm, 2, 0));         // E2: att' <- ctx
  T2_TRY(pack(m->w[W_DRNN_WIH], kdc, kARnn, 8, r_lstm, 2, 1));                //     dec <- ctx
  T2_TRY(pack(pk->wp_all, kdc, kDRnn, 8, r_p, 2, 2));                         //     P <- ctx
  T2_TRY(pack(m->w[W_DRNN_WHH], kDRnn, 0, 16, r_lstm, 3, 0));                 // E3: dec' <- dh
  T2_TRY(pack(pk->wp_all, kdc, 0, 16, r_p, 3, 1));                            //     P <- dh
  T2_TRY(pack(m->w[W_PRENET1], kPre, 0, 4, r_x2, 4, 0));                      // E4: x2 <- x1
  return T2_OK;
}

void persistent_pack_destroy(T2Model* m) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  if (!pk) return;
  cudaFree(pk->wimg); cudaFree(pk->plans); cudaFree(pk->wp_all); cudaFree(pk->bias_p);
  cudaFree(pk->bias_a); cudaFree(pk->bias_d); cudaFree(pk->rows); cudaFree(pk->weff); cudaFree(pk->weff_img);
  for (int i = 0; i < 2; ++i) cudaFree(pk->bwd_plans[i]);
  delete pk;
  m->pk = nullptr;
}

static int run_persistent_slice(T2Model* m, const T2DecoderArgs* a, cudaStream_t s, int b0, int nb);

int decoder_run_persistent(T2Model* m, const T2DecoderArgs* a, cudaStream_t s) {
  // batch rows are independent: more than 64 rows run as consecutive launches of <= 64 rows
  T2_CUDA(cudaMemsetAsync(a->n_steps, 0, sizeof(int32_t), s));
  for (int b0 = 0; b0 < a->B; b0 += kRows) {
    const int nb = a->B - b0 < kRows ? a->B - b0 : kRows;
    T2_TRY(run_persistent_slice(m, a, s, b0, nb));
  }
  return T2_OK;
}

// processed_memory = memory_layer(memory) of batch rows [b0, b0 + nb)                    (model.py:288)
static int processed_memory(T2Model* m, const T2DecoderArgs* a, int b0, int nb, float* pm, cudaStream_t s) {
  GemmArgs g;
  g.seg[0] = {a->memory + (size_t)b0 * a->T_enc * kEnc, kEnc, m->w[W_ATT_MEMORY], kEnc, kEnc};
  g.M = nb * a->T_enc; g.N = kAtt; g.C = pm; g.ldc = kAtt;
  return gemm_f32(g, s);
}

// the parameters of one launch over batch rows [b0, b0 + nb) that do not depend on where its state lives
static void slice_params(T2Model* m, const T2DecoderArgs* a, int b0, int nb, KParams* pp) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  KParams& p = *pp;
  const int T = a->T_enc, cap = a->n_steps_cap;
  memset(&p, 0, sizeof(p));
  p.plans = pk->plans; p.wimg = pk->wimg; p.bias_a = pk->bias_a; p.bias_d = pk->bias_d; p.bias_p = pk->bias_p;
  p.weff_img = pk->weff_img; p.w_v = m->w[W_ATT_V];
  p.memory = a->memory + (size_t)b0 * T * kEnc;
  p.mem_len = a->memory_lengths ? a->memory_lengths + b0 : nullptr;
  p.prenet_keep = a->prenet_keep; p.att_keep = a->att_keep; p.dec_keep = a->dec_keep;
  p.mel = a->mel + (size_t)b0 * cap * kMel; p.gate = a->gate + (size_t)b0 * cap; p.align = a->align + (size_t)b0 * cap * T;
  p.mel_lengths = a->mel_lengths + b0; p.n_steps = a->n_steps;
  p.b0 = b0; p.Btot = a->B;
  p.B = nb; p.T = T; p.cap = cap; p.infer = a->mode == T2_MODE_INFER; p.training = a->training;
  p.gate_threshold = a->gate_threshold; p.score_mask_value = a->score_mask_value;
  p.p_att = m->cfg.p_attention_dropout; p.p_dec = m->cfg.p_decoder_dropout; p.seed = a->seed;
  p.t_begin = 0; p.t_end = cap;
}

// x2 | ah | ctx | dh | x1 activation images, then q
static void carve_images(uint8_t* img, KParams* p) {
  p->x2_img = img; img += 4 * kXChunkBytes;
  p->ah_img = img; img += 16 * kXChunkBytes;
  p->ctx_img = img; img += 8 * kXChunkBytes;
  p->dh_img = img; img += 16 * kXChunkBytes;
  p->x1_img = img; img += 4 * kXChunkBytes;
  p->q = (float*)img;
}

// the longest T_enc that persistent_stages() runs with 4 stages (0 when none does); stages fall as T_enc grows
static int persistent_t4max() {
  if (persistent_stages(1) < 4) return 0;
  int lo = 1, hi = 1 << 16;                 // persistent_stages(lo) == 4, persistent_stages(hi) == 3
  while (hi - lo > 1) {
    const int mid = (lo + hi) / 2;
    if (persistent_stages(mid) == 4) lo = mid; else hi = mid;
  }
  return lo;
}

static int launch_persistent(KParams& p, cudaStream_t s) {
  p.nstages = persistent_stages(p.T);
  p.t4max = persistent_t4max();
  const size_t smem = persistent_smem_bytes(p.T, p.nstages);
  T2_CUDA(cudaFuncSetAttribute(decoder_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(kG); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeCooperative; attr.val.cooperative = 1;   // co-residency of all 128 CTAs
  cfg.attrs = &attr; cfg.numAttrs = 1;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, decoder_persistent_kernel, p);
  if (le != cudaSuccess) return fail(T2_ERR_CUDA, "persistent decoder launch failed: %s", cudaGetErrorString(le));
  if (getenv("T2_VERBOSE")) fprintf(stderr, "[t2b200] persistent decoder: B=%d T_enc=%d cap=%d stages=%d smem=%zu steps=%d-%d\n",
                                    p.B, p.T, p.cap, p.nstages, smem, p.t_begin, p.t_end);
  g_launch_count++;
  return T2_OK;
}

static int run_persistent_slice(T2Model* m, const T2DecoderArgs* a, cudaStream_t s, int b0, int nb) {
  const int T = a->T_enc, cap = a->n_steps_cap;
  DecoderWs w;
  T2_TRY(decoder_ws_carve(a, &w));
  T2_CUDA(cudaMemsetAsync(w.ctrl, 0, sizeof(DecoderCtrl), s));
  T2_CUDA(cudaMemsetAsync(w.images, 0, kImagesBytes, s));  // zero images (model.py:258-284)
  T2_TRY(processed_memory(m, a, b0, nb, w.pm, s));
  KParams p;
  slice_params(m, a, b0, nb, &p);
  carve_images(w.images, &p);
  p.pm = w.pm;
  p.ctrl = w.ctrl;
  const int B = nb;
  if (a->stash) {
    if (p.infer) return fail(T2_ERR_INVALID, "the training stash needs T2_MODE_TEACHER");
    if (a->stash_bytes < decoder_stash_bytes(a->B, cap)) return fail(T2_ERR_WORKSPACE, "decoder stash too small");
    Carve c(a->stash);
    decoder_stash_layout(c, a->B, cap, &p.st);
    if (b0 == 0) {   // slot 0 of the recurrent states = the zero initial states (model.py:258-284)
      float* z[5] = {p.st.ca, p.st.ha, p.st.cd, p.st.hd, p.st.ctx};
      for (int i = 0; i < 5; ++i)
        T2_CUDA(cudaMemsetAsync(z[i], 0, (size_t)a->B * (i < 4 ? kARnn : kEnc) * sizeof(float), s));
    }
  }
  if (!p.infer) {
    // teacher forcing (model.py:396-405): the prenet outputs of all steps are known up front -> convert
    // them once into x2 operand images, the kernel then skips the prenet events and their two barriers
    rows_to_image_kernel<<<dim3(4, cap), 256, 0, s>>>(a->teacher_prenet + (size_t)b0 * kPre, kPre, B, kPre, (long)a->B * kPre,
                                                      w.teacher_img, (long)4 * kXChunkBytes);
    T2_LAUNCH_CHECK();
    p.teacher_x2_img = w.teacher_img;
  }
  return launch_persistent(p, s);
}

// ---------------------------------------------------------------------------------------------
// resumable stream (t2_decoder_stream_*): every 64-row slice owns a block of the caller's state buffer
// ---------------------------------------------------------------------------------------------
struct StreamSlice {
  DecoderCtrl* ctrl;     // counters zeroed before every launch; the stop latch is carried in `done`
  uint8_t* images;       // activation images + q (kImagesBytes)
  float* acc; float* cell; float* att; int32_t* done;
  float* pm;             // processed memory of the slice's rows (nb, T, 128)
};
// the slices one after the other; returns slice `b0 / kRows` (any slice when only measuring)
__host__ __device__ static StreamSlice stream_state_layout(Carve& c, int B, int T, int b0) {
  const size_t tpp = (size_t)((T + kLocK - 1 + 3) & ~3);
  StreamSlice want = {};
  for (int b = 0; b < B; b += kRows) {
    const int nb = B - b < kRows ? B - b : kRows;
    StreamSlice sl;
    sl.ctrl = c.take<DecoderCtrl>(1, 1024);
    sl.images = c.take<uint8_t>(kImagesBytes, 1024);
    sl.acc = c.take<float>((size_t)kG * kRows * kAccPitch, 1024);
    sl.cell = c.take<float>((size_t)kG * 4 * kRows * 4, 1024);
    sl.att = c.take<float>((size_t)kG * 2 * tpp, 1024);
    sl.done = c.take<int32_t>(kRows, 1024);
    sl.pm = c.take<float>((size_t)nb * T * kAtt, 1024);
    if (b == b0) want = sl;
  }
  return want;
}
static StreamSlice stream_slice(void* state, int B, int T, int b0) { Carve c(state, 1024); return stream_state_layout(c, B, T, b0); }

size_t persistent_stream_state_bytes(int B, int T) { Carve c(nullptr, 1024); stream_state_layout(c, B, T, 0); return c.bytes(); }

int persistent_stream_begin(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, cudaStream_t s) {
  T2_CUDA(cudaMemsetAsync(state, 0, persistent_stream_state_bytes(a->B, a->T_enc), s));   // model.py:258-284
  T2_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * ((a->B + kRows - 1) / kRows), s));
  T2_CUDA(cudaMemsetAsync(a->mel_lengths, 0xff, sizeof(int32_t) * a->B, s));                // -1: still live
  T2_CUDA(cudaMemsetAsync(a->n_steps, 0, sizeof(int32_t), s));
  for (int b0 = 0; b0 < a->B; b0 += kRows)
    T2_TRY(processed_memory(m, a, b0, a->B - b0 < kRows ? a->B - b0 : kRows, stream_slice(state, a->B, a->T_enc, b0).pm, s));
  return T2_OK;
}

int persistent_stream_run(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, int n,
                          const int32_t* status_host, cudaStream_t s) {
  for (int b0 = 0, si = 0; b0 < a->B; b0 += kRows, ++si) {
    const int t0 = status_host ? status_host[2 * si] : 0;
    if ((status_host && status_host[2 * si + 1]) || t0 >= a->n_steps_cap) continue;    // this slice has stopped
    const StreamSlice sl = stream_slice(state, a->B, a->T_enc, b0);
    T2_CUDA(cudaMemsetAsync(sl.ctrl, 0, sizeof(DecoderCtrl), s));
    KParams p;
    slice_params(m, a, b0, a->B - b0 < kRows ? a->B - b0 : kRows, &p);
    carve_images(sl.images, &p);
    p.pm = sl.pm;
    p.ctrl = sl.ctrl;
    p.t_begin = t0;
    p.t_end = n < a->n_steps_cap - t0 ? t0 + n : a->n_steps_cap;
    p.rs_acc = sl.acc; p.rs_cell = sl.cell; p.rs_att = sl.att; p.rs_done = sl.done; p.rs_status = status + 2 * si;
    T2_TRY(launch_persistent(p, s));
  }
  return T2_OK;
}


// ---------------------------------------------------------------------------------------------
// continuous batching (t2_decoder_stream_admit / _collect): a stream whose rows are slots.  Between two chunks a row is
// put back to the state begin gives it and handed another text; after a chunk the frames of every occupied row go to
// the buffers of the request that holds it.
// ---------------------------------------------------------------------------------------------
namespace {
struct RowMask { uint64_t w[kMaxBatch / 64]; };      // bit b: row b is listed

// Block (r, slice) puts row r of its slice back to the state persistent_stream_begin leaves: zero is the initial value
// of every piece (model.py:258-284 starts both LSTMs, the attention weights and the context at zero, and an accumulator
// tile holds the partial products of zero activations).  It writes the row's own entries only.
__global__ void __launch_bounds__(256) stream_admit_kernel(void* state, int B, int T, RowMask mask, int32_t* mel_lengths) {
  const int lr = blockIdx.x, b0 = blockIdx.y * kRows, row = b0 + lr, tid = threadIdx.x;
  if (row >= B || !((mask.w[row >> 6] >> (row & 63)) & 1ull)) return;
  Carve c(state, 1024);
  const StreamSlice sl = stream_state_layout(c, B, T, b0);
  const int tpp = (T + kLocK - 1 + 3) & ~3;
  for (int i = tid; i < kG * kAccPitch; i += 256)                  // its accumulator row in every CTA's tile
    sl.acc[((size_t)(i / kAccPitch) * kRows + lr) * kAccPitch + i % kAccPitch] = 0.f;
  for (int i = tid; i < kG * 4; i += 256)                          // its cell states: (CTA, column group)
    reinterpret_cast<float4*>(sl.cell)[(size_t)i * kRows + lr] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = tid; i < 4 * tpp; i += 256)                         // previous | cumulative weights of CTAs lr and lr + 64
    sl.att[(size_t)(lr + 64 * (i / (2 * tpp))) * 2 * tpp + i % (2 * tpp)] = 0.f;
  for (int i = tid; i < kImageChunks * 2 * (kChunkK / 2); i += 256) {   // its row in both planes of every image chunk
    const int chunk = i / kChunkK, plane = (i / (kChunkK / 2)) & 1, k = (i % (kChunkK / 2)) * 2;
    __half* pl = reinterpret_cast<__half*>(sl.images + (size_t)chunk * kXChunkBytes) + plane * kRows * kChunkK;
    *reinterpret_cast<uint32_t*>(pl + img_elem_offset(lr, k)) = 0u;
  }
  float* q = reinterpret_cast<float*>(sl.images + (size_t)kImageChunks * kXChunkBytes);
  for (int i = tid; i < kAtt; i += 256) q[lr * kAtt + i] = 0.f;
  if (tid == 0) { sl.done[lr] = 0; mel_lengths[row] = -1; }
}

struct CollectBatch { T2CollectRow r[kRows]; int n; };   // the listed rows of one 64-row slice, by value

// block (t, i): frame t of the chunk buffers of row r[i].row -> frame t of that request's own buffers
__global__ void __launch_bounds__(128) stream_collect_kernel(const CollectBatch cb, const float* __restrict__ mel,
                                                             const float* __restrict__ gate, const float* __restrict__ align,
                                                             int cap, int T) {
  const T2CollectRow r = cb.r[blockIdx.y];
  const int t = blockIdx.x, tid = threadIdx.x;
  if (t >= r.n_frames) return;
  const size_t src = (size_t)r.row * cap + t;
  for (int i = tid; i < kMel; i += 128) r.mel[(size_t)t * kMel + i] = mel[src * kMel + i];
  if (tid == 0) r.gate[t] = gate[src];
  for (int i = tid; i < r.T_text; i += 128) r.align[(size_t)t * r.T_text + i] = align[src * T + i];
}
}  // namespace

int persistent_stream_admit(T2Model* m, const T2DecoderArgs* a, void* state, const int32_t* rows, int n_rows, cudaStream_t s) {
  RowMask mask;
  memset(&mask, 0, sizeof(mask));
  for (int i = 0; i < n_rows; ++i) mask.w[rows[i] >> 6] |= 1ull << (rows[i] & 63);
  stream_admit_kernel<<<dim3(kRows, (a->B + kRows - 1) / kRows), 256, 0, s>>>(state, a->B, a->T_enc, mask, a->mel_lengths);
  T2_LAUNCH_CHECK();
  // processed memory of the listed rows: one GEMM per run of consecutive rows of a slice (rows are ascending)
  for (int i = 0; i < n_rows;) {
    int j = i + 1;
    while (j < n_rows && rows[j] == rows[j - 1] + 1 && rows[j] / kRows == rows[i] / kRows) ++j;
    const int b0 = rows[i] / kRows * kRows;
    T2_TRY(processed_memory(m, a, rows[i], j - i, stream_slice(state, a->B, a->T_enc, b0).pm + (size_t)(rows[i] - b0) * a->T_enc * kAtt, s));
    i = j;
  }
  return T2_OK;
}

int persistent_stream_collect(const T2DecoderArgs* a, const T2CollectRow* rows, int n_rows, cudaStream_t s) {
  for (int b0 = 0; b0 < a->B; b0 += kRows) {
    CollectBatch cb;
    cb.n = 0;
    int frames = 0;
    for (int i = 0; i < n_rows; ++i)
      if (rows[i].row >= b0 && rows[i].row < b0 + kRows && rows[i].n_frames > 0) {
        cb.r[cb.n++] = rows[i];
        frames = rows[i].n_frames > frames ? rows[i].n_frames : frames;
      }
    if (cb.n == 0) continue;
    stream_collect_kernel<<<dim3(frames, cb.n), 128, 0, s>>>(cb, a->mel, a->gate, a->align, a->n_steps_cap, a->T_enc);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

#ifdef T2_SELFTEST
// ---------------------------------------------------------------------------------------------
// self test of the wgmma event engine: C (64 x N) = 2 * A (64 x K) . W (N x K)^T with the same run_event()
// (two accumulating passes over the ring) and the same accumulator tile as the decoder.  The N rows of W are
// the plan's consumers in order.
// ---------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(kThreads, 1)
selftest_kernel(const uint8_t* x_img, const uint8_t* w_img, EventPlan ep, int chunks, float* C, int N,
                DecoderCtrl* ctrl) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int tid = threadIdx.x;
  Carve sc(smem_raw, 1);
  GemmSmem sm;
  gemm_smem_layout(sc, &sm);
  Ring rg;
  rg.stage0 = sm.stage0;
  rg.full = sm.bars; rg.empty = sm.bars + kStages;
  float* s_acc = sm.acc;
  rg.p_stage = rg.p_phase = rg.c_stage = rg.c_phase = 0;
  rg.pol_x = rg.pol_w = ptx::policy_evict_last();
  rg.pre = 0; rg.ns = kStages;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { ptx::mbar_init(&rg.full[s], 1); ptx::mbar_init(&rg.empty[s], kMmaWgs); }
    ptx::fence_barrier_init();
  }
  for (int i = tid; i < kRows * kAccPitch; i += kThreads) s_acc[i] = 0.f;
  __syncthreads();
  run_event<true>(rg, ep, x_img, w_img, chunks, s_acc, ctrl, &ep);      // second pass uses the prefetched weights
  run_event<true>(rg, ep, x_img, w_img, chunks, s_acc, ctrl, nullptr);
  for (int i = tid; i < kRows * N; i += kThreads) C[i] = s_acc[(i / N) * kAccPitch + i % N];
}

// (N x K) fp32 row-major -> K/64 chunks of the plan's weight image (every consumer [n hi rows | n lo rows])
__global__ void pack_plan_image_kernel(const float* __restrict__ W, int K, EventPlan ep, uint8_t* __restrict__ wimg) {
  const int chunk = blockIdx.x;
  __half* img = reinterpret_cast<__half*>(wimg + (size_t)chunk * ep.w_bytes);
  for (int i = threadIdx.x; i < ep.nrows * 64; i += blockDim.x) {
    const int r = i >> 6, k = i & 63;
    int hr, lr;
    plan_image_rows(ep, r, hr, lr);
    __half h, l;
    split_fp16(W[(long)r * K + chunk * 64 + k], h, l);
    img[img_elem_offset(hr, k)] = h;
    img[img_elem_offset(lr, k)] = l;
  }
}

int selftest_plan(const float* A, const float* W, const EventPlan& ep, int K, float* C, cudaStream_t s) {
  const int chunks = K / kChunkK, N = ep.nrows;
  uint8_t *ximg = nullptr, *wimg = nullptr; DecoderCtrl* ctrl = nullptr;
  T2_CUDA(cudaMalloc((void**)&ximg, (size_t)chunks * kXChunkBytes));
  T2_CUDA(cudaMalloc((void**)&wimg, (size_t)chunks * ep.w_bytes));
  T2_CUDA(cudaMalloc((void**)&ctrl, sizeof(DecoderCtrl)));
  T2_CUDA(cudaMemsetAsync(ctrl, 0, sizeof(DecoderCtrl), s));
  rows_to_image_kernel<<<dim3(chunks, 1), 256, 0, s>>>(A, K, kRows, K, 0, ximg, 0);
  T2_LAUNCH_CHECK();
  pack_plan_image_kernel<<<chunks, 256, 0, s>>>(W, K, ep, wimg);
  T2_LAUNCH_CHECK();
  const size_t smem = gemm_smem_bytes();
  T2_CUDA(cudaFuncSetAttribute(selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  selftest_kernel<<<1, kThreads, smem, s>>>(ximg, wimg, ep, chunks, C, N, ctrl);
  T2_LAUNCH_CHECK();
  T2_CUDA(cudaStreamSynchronize(s));
  cudaFree(ximg); cudaFree(wimg); cudaFree(ctrl);
  return T2_OK;
}
}  // namespace

int selftest_umma(const float* A, const float* W, int N, int K, int passes, float* C, cudaStream_t s) {
  (void)passes;
  if (N % 8 != 0 || N < 8 || N > kHiCols || K % kChunkK != 0 || K <= 0)
    return fail(T2_ERR_INVALID, "selftest_umma: N in {8..80 step 8}, K %% 64 == 0");
  EventPlan ep; memset(&ep, 0, sizeof(ep));
  plan_one_matrix(ep, N);
  ep.chunks = K / kChunkK;
  return selftest_plan(A, W, ep, K, C, s);
}

int selftest_event(const float* A, const float* W, const int* cons, int ncons, int K, float* C, cudaStream_t s) {
  EventPlan ep; memset(&ep, 0, sizeof(ep));
  if (ncons < 1 || ncons > 3 || K % kChunkK != 0 || K <= 0 || K > 16 * kChunkK)
    return fail(T2_ERR_INVALID, "selftest_event: 1-3 consumers, K a multiple of 64 up to 1024");
  for (int i = 0; i < ncons; ++i) { ep.n[i] = cons[i]; ep.nrows += cons[i]; }
  ep.ncons = ncons; ep.w_bytes = (uint32_t)ep.nrows * 256; ep.chunks = K / kChunkK;
  if (!event_plan_fits(ep, true))
    return fail(T2_ERR_INVALID, "selftest_event: 1-3 consumers of 8, 16, 24 or 32 rows");
  return selftest_plan(A, W, ep, K, C, s);
}

#endif  // T2_SELFTEST

// ---------------------------------------------------------------------------------------------
// Backward skinny GEMMs of the training path on the tensor cores (decoder_backward.cu, KB / KE):
//   P[split][b][col] = inv_scale[b] * sum_{n in the split's chunks} dG_scaled[b][n] * Wcat[n][col]
// dG (64 x 4096) arrives as a split-fp16 activation image whose rows were scaled by a power of two
// (row maximum in [0.5, 1): gradients span many orders of magnitude, fp16 does not); Wcat = [W_ih | W_hh]
// is streamed as W^T images (rows = output columns, K = gate rows).  Same ring / MMA / accumulator tile
// as the forward events (run_event): a tile of output columns is planned as consumers of 32, 32 and 16 columns.
// ---------------------------------------------------------------------------------------------
namespace {
constexpr int kBwdTileB = 80, kBwdTileE = 64;       // output columns per CTA: 2560 = 32 x 80, 1792 = 28 x 64

__global__ void pack_bwd_wimg_kernel(const float* __restrict__ w0, int cols0, const float* __restrict__ w1, int cols1,
                                     const BwdCta* __restrict__ plans, uint8_t* __restrict__ wimg) {
  // grid (max chunks per CTA, n_cta): image block of chunk j of CTA c: rows = its output columns, k = 64 gate rows
  const BwdCta& pc = plans[blockIdx.y];
  const int j = blockIdx.x;
  if (j >= pc.nchunks) return;
  const int n = pc.ep.nrows;
  __half* img = reinterpret_cast<__half*>(wimg + pc.ep.w_off + (size_t)j * pc.ep.w_bytes);
  const int n0 = (pc.chunk0 + j) * kChunkK;
  for (int i = threadIdx.x; i < n * kChunkK; i += blockDim.x) {
    const int k = i / n, r = i - k * n;            // r fastest: coalesced along the weight matrix' columns
    const int col = pc.col0 + r;
    const float v = col < cols0 ? w0[(long)(n0 + k) * cols0 + col] : w1[(long)(n0 + k) * cols1 + (col - cols0)];
    int hr, lr;
    plan_image_rows(pc.ep, r, hr, lr);
    __half h, l;
    split_fp16(v, h, l);
    img[img_elem_offset(hr, k)] = h;
    img[img_elem_offset(lr, k)] = l;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
bwd_gemm_kernel(const uint8_t* __restrict__ x_img, const uint8_t* __restrict__ w_img, const BwdCta* __restrict__ plans,
                const float* __restrict__ inv_scale, float* __restrict__ P, int ldp, DecoderCtrl* ctrl) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int tid = threadIdx.x;
  const BwdCta pc = plans[blockIdx.x];
  Carve sc(smem_raw, 1);
  GemmSmem sm;
  gemm_smem_layout(sc, &sm);
  Ring rg;
  rg.stage0 = sm.stage0;
  rg.full = sm.bars; rg.empty = sm.bars + kStages;
  float* s_acc = sm.acc;
  rg.p_stage = rg.p_phase = rg.c_stage = rg.c_phase = 0;
  rg.pol_x = ptx::policy_evict_last(); rg.pol_w = ptx::policy_evict_first();
  rg.pre = 0; rg.ns = kStages;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { ptx::mbar_init(&rg.full[s], 1); ptx::mbar_init(&rg.empty[s], kMmaWgs); }
    ptx::fence_barrier_init();
  }
  for (int i = tid; i < kRows * kAccPitch; i += kThreads) s_acc[i] = 0.f;
  __syncthreads();
  run_event(rg, pc.ep, x_img + (size_t)pc.chunk0 * kXChunkBytes, w_img, pc.nchunks, s_acc, ctrl, nullptr);
  const int N = pc.ep.nrows;
  for (int i = tid; i < kRows * N; i += kThreads) {
    const int row = i / N, c = i - row * N;
    P[((size_t)pc.split * kRows + row) * ldp + pc.col0 + c] = s_acc[row * kAccPitch + c] * inv_scale[row];
  }
}

}  // namespace

int bwd_gemm_ctas(int which) { return which == 0 ? (2560 / kBwdTileB) * kBwdGemmSplit : (1792 / kBwdTileE) * kBwdGemmSplit; }

namespace {
constexpr int kBwdChunks = 4 * kARnn / kChunkK;                   // 64 K chunks
int bwd_tile(int which) { return which == 0 ? kBwdTileB : kBwdTileE; }
uint32_t bwd_w_bytes(int which) { return (uint32_t)(2 * bwd_tile(which) * kChunkK * 2); }

std::vector<BwdCta> bwd_gemm_plans(int which) {
  const int tile = bwd_tile(which), ntile = (which == 0 ? 2560 : 1792) / tile;
  const uint32_t w_bytes = bwd_w_bytes(which);
  std::vector<BwdCta> plans(ntile * kBwdGemmSplit);
  for (int t = 0; t < ntile; ++t)
    for (int sp = 0; sp < kBwdGemmSplit; ++sp) {
      BwdCta& c = plans[t * kBwdGemmSplit + sp];
      memset(&c, 0, sizeof(c));
      c.chunk0 = sp * kBwdChunks / kBwdGemmSplit; c.nchunks = (sp + 1) * kBwdChunks / kBwdGemmSplit - c.chunk0;
      c.col0 = t * tile; c.split = sp;
      plan_one_matrix(c.ep, tile);    // 80 = 32 + 32 + 16, 64 = 32 + 32 columns (event_plan_fits(c.ep, false))
      c.ep.col0 = 0; c.ep.chunks = c.nchunks;
      c.ep.w_off = (uint32_t)(((size_t)t * kBwdChunks + c.chunk0) * w_bytes);
    }
  return plans;
}
}  // namespace

size_t bwd_wimg_bytes(int which) { return (size_t)((which == 0 ? 2560 : 1792) / bwd_tile(which)) * kBwdChunks * bwd_w_bytes(which); }

// packs the W^T images of both LSTMs from the caller's current fp32 weights into wimg[0 / 1] (bwd_wimg_bytes)
int bwd_gemm_prepare(T2Model* m, uint8_t* const* wimg, cudaStream_t s) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  if (!pk) return fail(T2_ERR_INVALID, "backward GEMM: model has no persistent pack");
  for (int which = 0; which < 2; ++which) {
    const float* w0 = m->w[which == 0 ? W_DRNN_WIH : W_ARNN_WIH];
    const float* w1 = m->w[which == 0 ? W_DRNN_WHH : W_ARNN_WHH];
    const int cols0 = which == 0 ? kARnn + kEnc : kPre + kEnc;
    pack_bwd_wimg_kernel<<<dim3(kBwdChunks / kBwdGemmSplit, bwd_gemm_ctas(which)), 256, 0, s>>>(w0, cols0, w1, kARnn,
                                                                                             pk->bwd_plans[which], wimg[which]);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

int bwd_gemm_run(T2Model* m, int which, const uint8_t* w_img, const uint8_t* x_img, const float* inv_scale, float* P, int ldp,
                 DecoderCtrl* ctrl, cudaStream_t s) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  const size_t smem = gemm_smem_bytes();
  T2_CUDA(cudaFuncSetAttribute(bwd_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  bwd_gemm_kernel<<<bwd_gemm_ctas(which), kThreads, smem, s>>>(x_img, w_img, pk->bwd_plans[which], inv_scale, P, ldp, ctrl);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
