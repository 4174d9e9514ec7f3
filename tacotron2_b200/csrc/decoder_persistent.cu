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
//        ah_t  -> dec gates += W_ih^d[:, :1024] ah ; q = W_q ah
//        ah_t  -> att gates(t+1) += W_hh^a ah   (Ed: CTA c < 64 streams it for itself and for CTA c + 64 during the
//                                                attention, which CTA c + 64 runs)
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
//     weights (kept in shared memory across steps); energies, softmax and context of batch row b on CTA b + 64
//     with warp-shuffle reductions.
//   * events are separated by a grid-wide barrier or by producer-scoped counters (monotonic global counters:
//     fence.acq_rel + relaxed red to arrive, relaxed polls + one fence to wait).
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "decoder.h"
#include "event_engine.cuh"
#include "gemm_f32.cuh"

namespace t2 {

namespace {

constexpr int kG = 128;               // CTAs
constexpr int kMaxStages = 4;          // the decoder kernel runs 4 stages up to T_enc = 896, else 3
                                       // (T2_STAGES = 3 forces the 3-stage ring)
// accumulator columns (shared memory, fp32 [64 batch rows][kAccPitch]): att 0-31, dec 32-63, shared slot 64-79
constexpr int kColA = 0, kColD = 32, kColS = 64;
constexpr int kAttRound = 64;                             // encoder positions per attention pa GEMM
constexpr int kAttPlane = kAttRound * 128;                // one fp16 plane of the im2col image (64 positions x 64 taps)
constexpr int kPaPitch = kAttRound + 4;                   // floats per attention dim of the pa tile
constexpr int kPaBytes = kAtt * kPaPitch * 4;
constexpr int kNumEvents = 6;         // x2, ah, ctx, dh, x1, deferred ah (Ed)
constexpr int kEd = 5;
constexpr int kPCols = 344;           // 80 mel + 1 gate + 256 x1 + 7 pad
constexpr int kQCta0 = 0, kQCtas = 16, kX2Cta0 = 16, kX2Ctas = 32, kPCta0 = 48, kPCtas = 43;
constexpr int kAttCta0 = 64;          // CTA kAttCta0 + b runs the attention of batch row b
// Ed waits for the query counter (true) or starts right after E1, with its first weight chunks prefetched by E1 (false):
// the query CTAs stream E1 without the deferred stream's HBM traffic, or Ed gets the longer window.  Both ran the decoder
// step in 65.4-66.0 µs on an H100 at 700 W (DESIGN §6.1).
constexpr bool kEdAfterQ = true;
constexpr int kWeffBytes = kAtt * kChunkK * 2 * 2;        // fused location filter image (hi+lo) = 32 KiB

struct CtaPlan {
  EventPlan ev[kNumEvents];
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
};

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

// consumer cons + blockIdx.z of one event: for CTA blockIdx.y, chunk blockIdx.x: rows rows_tab[z*tab_stride + cta*32 + i]
// (-1 = zero row) x 64 columns starting at kcol0 + chunk*64 go to rows [roff, roff+n) of the chunk's hi and lo planes
// (each plane holds the rows of ALL consumers of the event, concatenated).
__global__ void pack_consumer_kernel(const float* __restrict__ src, int ld, int kcol0,
                                     const int32_t* __restrict__ rows_tab, int tab_stride, const CtaPlan* __restrict__ plans,
                                     int ev, int cons, uint8_t* __restrict__ wimg) {
  const int cta = blockIdx.y, chunk = blockIdx.x;
  cons += blockIdx.z;
  rows_tab += blockIdx.z * tab_stride;
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

}  // namespace

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

namespace {

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
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

// floats of a padded attention-weight row: T_enc + the location conv's kLocK - 1 zero taps, rounded up to whole float4
__host__ __device__ constexpr int att_pad_len(int T) { return (T + kLocK - 1 + 3) & ~3; }

// Dynamic shared memory of the persistent decoder for (T_enc, ring stages): the kernel carves it and the host sizes
// the launch from it, which decides the ring depth and the longest T_enc.  The regions are packed in this order.
struct PersistentSmem {
  uint8_t* stage0;                 // ring stages
  uint8_t* weff;                   // fused location filter image
  float* acc;                      // event accumulators
  uint64_t* bars;                  // 16 slots: full[kMaxStages] | empty[kMaxStages] | pa tile
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
  const int tpp = att_pad_len(T), ntiles = (T + 127) >> 7;
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
  // activation images, q and pa: the launch's slice block (SliceState, host side); pm: rows b0.. of the buffer's (B, T, 128)
  uint8_t* x2_img; uint8_t* ah_img; uint8_t* ctx_img; uint8_t* dh_img; uint8_t* x1_img;
  const uint8_t* teacher_x2_img;   // (cap, 4 chunks) or null
  float* q;                         // (64, 128) fp32
  float* part;                      // (64 lower CTAs, 64, 32) fp32: W_hh^a . ah_t of CTA c + 64's units, from CTA c's Ed
  float* pa;                        // (64, 128, pa_pitch(T)) fp32 location term of the next step; null: computed in the
                                    // attention phase (TEACHER, or a tile that does not fit the ring)
  float* mel; float* gate; float* align; int32_t* mel_lengths; int32_t* n_steps;
  DecoderCtrl* ctrl;
  int B, T, cap, infer, training;
  int nstages;                      // operand ring stages (4, or 3 when T_enc > 896)
  int t4max;                        // longest T_enc that runs with 4 stages (0: every T_enc runs with 3)
  int b0, Btot;                     // this launch handles batch rows [b0, b0 + B) of Btot (dropout mask / Philox indexing)
  float gate_threshold, score_mask_value, p_att, p_dec;
  uint64_t seed;
  // per-row prenet keys (INFER; row_seeds == nullptr: p.seed and element (b0 + row) * 256 + column): row r draws with
  // key row_seeds[b0 + r], element = column, at its own step row_step0[b0 + r] + t (row_step0 == nullptr: t).  Read from
  // global memory at the draw: a table in shared memory would cost the 3-stage layout its longest T_enc.
  const uint64_t* row_seeds; const int32_t* row_step0;
  DecoderStash st;                  // training stash for the backward pass (st.ga == nullptr: none)
  int t_begin, t_end;               // this launch runs steps [t_begin, t_end); the whole loop: 0, cap
  // resumable stream (t2_decoder_stream_run; rs_acc == nullptr: none).  The prologue restores and the epilogue saves the
  // on-chip state that lives past a step boundary, in the saved part of the slice block; the activation images, q, pa and
  // the processed memory stay in place.
  float* rs_acc;                    // (kG, kRows x kAccPitch) accumulator tiles: next-step partial products
  float* rs_cell;                   // (kG, 4 column groups, kRows) float4 {c_att[0], c_att[1], c_dec[0], c_dec[1]}
  float* rs_att;                    // (64 attention CTAs, 2, padded TP) previous | cumulative attention weights
  int32_t* rs_done;                 // (kRows) stop latch
  int32_t* rs_status;               // out: [steps run, stopped]
  // forced alignment (INFER, the kForced instantiation): rows b0.. of the given attention weights (Btot, cap, T) and
  // their step counts (Btot), clamped into [1, cap] where they are read
  const float* forced_align; const int32_t* forced_lengths;
  // limits (INFER, the kLimited instantiation; win_front == 0: the other two): at step t row r attends only to
  // [p - win_back, p + win_front), p = the first argmax of its previous weights below its length, and with max_steps
  // (rows b0.. of (Btot), clamped into [1, cap] where they are read) it stops after max_steps[r] steps at the latest
  int win_back, win_front; const int32_t* max_steps;
};

// The context's grouping of a T_enc-long row: the half rows (256 columns) of encoder memory that an idle ring of `nstages`
// stages holds beside the im2col image and one round's pa tile.  The context of a row sums its positions split there, in
// the grouping a launch sized for that row's own length uses (see the context below), wherever its rows actually live:
// the attention CTA stages fewer whole rows and reads the rest from L2.
__host__ __device__ constexpr int staged_rows(int T, int nstages) {
  return T < (nstages * kStageBytes - 2 * kAttPlane - kPaBytes) / (kEnc / 2 * 4)
             ? T : (nstages * kStageBytes - 2 * kAttPlane - kPaBytes) / (kEnc / 2 * 4);
}

// INFER precomputes the location term pa of step t+1 during the x2 wait of step t (see the kernel) into a global buffer of
// one fp32 tile [128 dims][pa_pitch(T)] per batch row.  The pitch covers the energies' last chunk of 8 positions, and it is
// an odd number of 16-byte units (whole units for the bulk copy; odd so that the float4 reads of 8 consecutive dims at one
// position hit distinct banks).
__host__ __device__ constexpr int pa_pitch(int T) { return ((T + 7) & ~7) + 4; }
__host__ __device__ constexpr int pa_tile_bytes(int T) { return kAtt * pa_pitch(T) * 4; }
// The whole tile is copied into the idle ring before the q barrier, so it must fit there: T_enc <= 280 at 4 stages (<= 208
// with 3 stages forced; the 3-stage layout otherwise only runs T_enc > 896).  Longer memories compute pa after the q
// barrier round by round, as TEACHER does.
__host__ __device__ constexpr bool pa_tile_fits(int T, int nstages) { return pa_tile_bytes(T) <= nstages * kStageBytes; }

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
// kModeForced (INFER with p.forced_align): the attention weights of step t are row t of the given map instead of the
// softmax of the energies, and row b stops after forced_lengths[b] steps instead of on its gate.  The location term, the
// energies and the softmax are skipped; the events, barriers and the context routine are those of the free run.
// kModeLimited (INFER with limits): the free run, with the energies outside the row's attention window masked before the
// softmax and a stop latch that also fires at the row's own step limit.  Everything else is the free run's.
enum : int { kModeFree = 0, kModeForced = 1, kModeLimited = 2 };
template <int kMode>
__global__ void __launch_bounds__(kThreads, 1) decoder_persistent_kernel(const KParams p) {
  constexpr bool kForced = kMode == kModeForced, kLimited = kMode == kModeLimited;
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

  uint64_t* bar_pa = sm.bars + 2 * kMaxStages;   // bulk copy of this step's pa tile
  uint32_t pa_phase = 0;
  if (tid == 0) {
    for (int s = 0; s < p.nstages; ++s) { ptx::mbar_init(&rg.full[s], 1); ptx::mbar_init(&rg.empty[s], kMmaWgs); }
    ptx::mbar_init(bar_pa, 1);
    ptx::fence_barrier_init();
  }
  const bool resume = p.rs_acc != nullptr;       // a stream's chunk: its state was zeroed by begin or saved by the last chunk
  const int tpp = att_pad_len(T);
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
  // the previous / cumulative attention weights live on the attention CTAs kAttCta0.. (model.py:274-277)
  const bool upper = cta >= kAttCta0;
  for (int i = tid; i < TP; i += kThreads) {
    s_pad0[i] = resume && upper ? p.rs_att[((size_t)(cta - kAttCta0) * 2 + 0) * tpp + i] : 0.f;
    s_pad1[i] = resume && upper ? p.rs_att[((size_t)(cta - kAttCta0) * 2 + 1) * tpp + i] : 0.f;
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
  // this thread's saved cell states (resume); recomputed where it is used, so that no pointer stays live across the loop
  auto rs_cell = [&]() { return reinterpret_cast<float4*>(p.rs_cell) + ((size_t)cta * 4 + cg) * kRows + row; };
  if (resume && !is_lo) {
    const float4 c = *rs_cell();
    c_att[0] = c.x; c_att[1] = c.y; c_dec[0] = c.z; c_dec[1] = c.w;
  }
  const bool has_q = cta >= kQCta0 && cta < kQCta0 + kQCtas;
  const bool has_x2 = cta >= kX2Cta0 && cta < kX2Cta0 + kX2Ctas;
  const int halfk = (kLocK - 1) / 2;
  // phase profile (cycles, accumulated over steps) on three sample CTAs; see t2_decoder_profile().  The limited
  // instantiation keeps none: its clock registers would push the window's argmax over 128 registers into spills.
  const int prof_slot = kLimited ? -1 : cta == 0 ? 0 : (cta == 60 ? 1 : (cta == 100 ? 2 : -1));
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
        // Philox key, step and the row's first element: one stream per call (b0 + row) * 256 + column, or per row
        uint64_t seed = p.seed, e0 = (uint64_t)(p.b0 + row) * kPre;
        uint32_t step = t + 1;
        if (p.row_seeds) {
          seed = p.row_seeds[p.b0 + row];
          e0 = 0;
          if (p.row_step0) step += p.row_step0[p.b0 + row];
        }
        if (has_x2) {
          const int col0 = (cta - kX2Cta0) * 8;
          if (p.prenet_keep) {
            const uint8_t* kp = p.prenet_keep + ((long)(t + 1) * 2 + 1) * p.Btot * kPre + (long)(p.b0 + row) * kPre + col0;
            for (int j = 0; j < 8; ++j) bits |= (kp[j] != 0 ? 1u : 0u) << j;
          } else {
            bits = philox_keep8(seed, step * 4 + 1, e0 + col0, 0.5f);
          }
        } else {
          const int pc0 = (cta - kPCta0) * 8;
          for (int j = 0; j < 8; ++j) {
            const int col = pc0 + j - (kMel + 1);
            if (col < 0 || col >= kPre) continue;
            const long idx = (long)(p.b0 + row) * kPre + col;
            const bool keep = p.prenet_keep ? p.prenet_keep[((long)(t + 1) * 2 + 0) * p.Btot * kPre + idx] != 0
                                            : philox_keep(seed, step * 4 + 0, e0 + col, 0.5f);
            bits |= (keep ? 1u : 0u) << j;
          }
        }
        s_mask[row] = bits;
      }
      // the attention phase reuses the ring of an upper CTA as scratch; a lower one goes on with Ed
      run_event(rg, plan.ev[1], p.ah_img, p.wimg, 16, s_acc, ctrl, upper || kEdAfterQ ? nullptr : &plan.ev[kEd],
                ctrl->ah_count, 8u * (unsigned int)(t + 1 - p.t_begin));
      if (has_q) {
        if (cg == 0 && !is_lo) {
          float g[8];
          acc_take8(s_acc, row, kColS, 0, g);
          if (erow) {
#pragma unroll
            for (int j = 0; j < 8; ++j) p.q[row * kAtt + (cta - kQCta0) * 8 + j] = g[j];
          }
        }
        signal_counter(&ctrl->q_count, 1u);                                  // B2: this CTA's 8 columns of q are written
      }
      T2_PROF(3);
    }
    // ======== Ed: ah_t -> att gates(t+1) += W_hh^a ah of this CTA's units and of its partner's (CTA + 64) ========
    // The lower CTAs stream it while the upper ones run the attention; E1 acquired every ah chunk.  The partner's sums go
    // to p.part and are added to its tile after B3, ahead of E2, as the first term of those columns (they are zero before
    // it), so the addition order is the one of a single event.  Every lower CTA runs it: its units exist at any B.
    if (!upper) {
      if (kEdAfterQ) {
        wait_counter(&ctrl->q_count, (unsigned int)(kQCtas * (t + 1 - p.t_begin)), s_flag, ctrl, 105);
        T2_PROF(4);
      }
      run_event(rg, plan.ev[kEd], p.ah_img, p.wimg, 16, s_acc, ctrl, &plan.ev[2], nullptr, 0,
                p.part + (size_t)cta * kRows * 32);
      T2_PROF(21);
    }
    // ======== attention for batch row b = cta - kAttCta0 ======================= model.py:43-86, 358-365
    // CTA b+64 evaluates row b's energies, softmax, alignment row and all 512 context columns; CTA b keeps its ring for
    // the deferred event Ed below.  Everything that only needs THIS CTA's state (the pa tile, staging encoder memory
    // rows) runs between the arrival at barrier B2 and the wait for it.
    // The location term pa of step t depends only on the attention weights of step t-1.  With p.pa (INFER, tile fits the
    // ring) the attention CTA computes it during the x2 wait of step t-1, when its ring is idle, and bulk-copies the whole
    // tile before B2; after B2 the energies are one pass over all positions.  Otherwise (TEACHER: no x2 wait, the ring
    // holds the prefetched E0 weights; or a T_enc whose tile does not fit) pa is computed here, 64 positions per round,
    // round 0 before the B2 wait.
    const bool att_cta = upper && cta - kAttCta0 < p.B;
    const int att_b = cta & 63;
    const bool pa_pre = !kForced && p.pa != nullptr;
    const int pa_p = pa_pitch(T);
    float* pa_row = pa_pre ? p.pa + (size_t)att_b * kAtt * pa_p : nullptr;
    uint8_t* aimg = rg.stage0;
    // the idle operand ring during the attention phase: [im2col image: hi plane | lo plane][pa tile of one round]
    // [encoder-memory rows], or with p.pa [pa tile of all positions][encoder-memory rows]
    const int att_rounds = (T + kAttRound - 1) / kAttRound;
    const int img_bytes = 2 * kAttPlane;
    float* s_pa = reinterpret_cast<float*>(aimg + img_bytes);                       // [128 dims][kPaPitch] fp32
    const int mem_off = pa_pre ? pa_tile_bytes(T) : img_bytes + kPaBytes;         // ring bytes before the memory rows
    const int smem_rows = min(T, (p.nstages * kStageBytes - mem_off) / (kEnc * 4));   // memory rows staged in the ring
    // pa^T = Weff . A^T on the tensor cores (fused model.py:23-25), i.e. the fused filter bank is the M = 128 operand
    // (attention dim d; warpgroups 0 / 1 take dims 0-63 / 64-127) and kAttRound positions are the N dimension.  The
    // tile of round r0 goes to dst[dim * pitch + position - 64 r0] (positions below `bound`): in shared memory every warp
    // then owns a slice of POSITIONS of all 128 dims, so the tanh of a row spread evenly over the four SM sub-partitions
    // for any T_enc, the processed-memory reads are coalesced (lanes = consecutive dims) and can be issued before the q
    // barrier.
    auto att_pa_round = [&](int r0, float* dst, int pitch, int bound) {
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
        for (int i = 0; i < kAttRound / 2; i += 2) {
          const int col = ptx::wg_frag_col(i, wt);
          float* o = dst + (wg * 64 + ptx::wg_frag_row(i, wt)) * pitch + col;
          if (col + 1 < bound) *reinterpret_cast<float2*>(o) = make_float2(d[i], d[i + 1]);
          else if (col < bound) *o = d[i];
        }
      }
      __syncthreads();
    };
    auto stage_memory_rows = [&](int j0, int j1) {     // cp.async memory rows [j0, j1) into the ring
      const uint32_t sbase = ptx::smem_u32(rg.stage0) + (uint32_t)mem_off;
      const float* msrc = p.memory + (long)att_b * T * kEnc;
      for (int i = j0 * (kEnc / 4) + tid; i < j1 * (kEnc / 4); i += kThreads) {
        const int j = i >> 7, c4 = i & 127;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sbase + (uint32_t)i * 16u),
                     "l"(msrc + (long)j * kEnc + c4 * 4)
                     : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const int adim = quad * 32 + lane;     // this thread's attention dim
    float pm_next[8];                      // processed-memory values of the thread's next chunk of 8 positions (software pipeline)
    auto load_pm = [&](const float* pmr, int j0, int cnt) {
#pragma unroll
      for (int e = 0; e < 8; ++e) pm_next[e] = (j0 + e < cnt) ? __ldg(pmr + (long)(j0 + e) * kAtt) : 0.f;
    };
    if (att_cta && kForced) {
      // the weights of step t do not depend on q: row t of the row's map (zero past its text length, and all zero once
      // the row has run its steps, without reading the map) goes to s_e and the alignment output before the q barrier
      const int len = p.mem_len ? min(p.mem_len[att_b], T) : T;
      const int flen = min(max(p.forced_lengths[att_b], 1), p.cap);
      const float* fa = p.forced_align + ((long)att_b * p.cap + t) * T;
      for (int j = tid; j < T; j += kThreads) {
        const float a = (t < flen && j < len) ? __ldg(fa + j) : 0.f;
        s_e[j] = a;
        p.align[((long)att_b * p.cap + t) * T + j] = a;
      }
      stage_memory_rows(0, smem_rows);
    } else if (att_cta) {
      if (pa_pre) {
        // this CTA wrote the tile before it signalled its ah columns of this step (which fences it for the async
        // proxy), or in the launch of the previous chunk, or the buffer was zeroed before step 0 (the attention weights
        // start at zero, so pa is +0.0)
        if (tid == 0) {
          ptx::mbar_arrive_expect_tx(bar_pa, (uint32_t)pa_tile_bytes(T));
          ptx::bulk_g2s_hint(rg.stage0, pa_row, (uint32_t)pa_tile_bytes(T), bar_pa, rg.pol_w);
        }
      } else {
        att_pa_round(0, s_pa, kPaPitch, kAttRound);
      }
      stage_memory_rows(0, smem_rows);     // everything the context needs is in flight before the q barrier
      load_pm(p.pm + (long)att_b * T * kAtt + adim, cg * 8, min(T, kAttRound));
    }
    T2_PROF(15);
    if (att_cta) wait_counter(&ctrl->q_count, (unsigned int)(kQCtas * (t + 1 - p.t_begin)), s_flag, ctrl, 104);   // B2
    T2_PROF(4);
    if (att_cta) {
      const int b = att_b;
      if constexpr (!kForced) {             // the query, the location term and the energies
        for (int i = tid; i < kAtt; i += kThreads) s_q[i] = __ldcg(&p.q[b * kAtt + i]);
        __syncthreads();
        {
          const int eN = ntiles * 128;
          const float qd = s_q[adim], vd = s_v[adim];
          // with the copied tile: one pass over all T positions; else one round of 64 positions per pa GEMM.  Chunks of 8
          // positions start at multiples of 8 either way, so every energy is the same sum in the same order.
          const int nrounds = pa_pre ? 1 : att_rounds, rlen = pa_pre ? T : kAttRound;
          const float* s_tile = pa_pre ? reinterpret_cast<const float*>(rg.stage0) : s_pa;
          const int tpitch = pa_pre ? pa_p : kPaPitch;
          if (pa_pre) { mbar_wait(bar_pa, pa_phase, ctrl, 207); pa_phase ^= 1; }
          for (int r0 = 0; r0 < nrounds; ++r0) {
            const int jbase = r0 * kAttRound, cnt = min(T - jbase, rlen), nch = (cnt + 7) >> 3;
            if (r0 > 0) att_pa_round(r0, s_pa, kPaPitch, kAttRound);
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
                const float4 g0 = *reinterpret_cast<const float4*>(s_tile + adim * tpitch + j0);
                const float4 g1 = *reinterpret_cast<const float4*>(s_tile + adim * tpitch + j0 + 4);
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
      }
      // mask + softmax (model.py:79-82): every warp reduces all T energies itself (shuffles only, no
      // cross-warp exchange), then the threads split the normalised write-out
      const int len = p.mem_len ? min(p.mem_len[b], T) : T;
      if constexpr (!kForced) {             // the softmax and the previous / cumulative weights
        const int eN = ntiles * 128;
        // the attention window [wlo, whi) of this step: p_t is the first position of the largest previous weight below
        // len (0 while they are all zero).  Every warp reduces it itself from the previous weights, which the write-out
        // below overwrites only after the barrier that follows the mask.
        // The weights are >= +0.0 (softmax outputs, or the zeros of begin / admit), so their bit patterns order as their
        // values: one integer max reduction, then one min reduction over the first position of each lane that holds it.
        int wlo = 0, whi = len;
        if constexpr (kLimited) {
          unsigned bv = 0u;
          for (int j = lane; j < len; j += 32) bv = max(bv, __float_as_uint(s_pad0[halfk + j]));
          bv = __reduce_max_sync(0xffffffffu, bv);
          unsigned bj = (unsigned)len;
          for (int j = lane; j < len; j += 32)
            if (__float_as_uint(s_pad0[halfk + j]) == bv) { bj = (unsigned)j; break; }
          const int pt = (int)__reduce_min_sync(0xffffffffu, bj);
          wlo = pt - p.win_back;
          whi = min(len, pt + p.win_front);
        }
        // masked energies once (the four 32-dim partial sums added in a fixed order), in place in the first partial-sum plane
        for (int j = tid; j < T; j += kThreads)
          s_ep[j] = (kLimited ? (j >= wlo && j < whi) : j < len)
                        ? (s_ep[j] + s_ep[eN + j]) + (s_ep[2 * eN + j] + s_ep[3 * eN + j]) : p.score_mask_value;
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
          p.align[((long)b * p.cap + t) * T + j] = a;
        }
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      T2_PROF(18);
      {                                                           // context = aw . memory  model.py:83-84
        // j-group jg sums positions jg, jg + 8, ... below `split`, then split + jg, split + jg + 8, ... below `clen`.
        // INFER: clen = len and split = the rows a launch sized for T_enc = len stages, so the grouping is a function of
        // the row's own length, not of the launch's T_enc, and a row of a ragged batch gets the bits it gets alone
        // (positions >= len have weight 0 and are skipped).  Without lengths, len = T_enc and split = staged_rows(T_enc).
        // TEACHER keeps the launch's grouping over all T_enc positions.  `split` counts half rows of 256 columns, as the
        // ring of a CTA pair that split the columns staged them, so the grouping is not where a row lives: the ring holds
        // fewer of the whole 512-column rows, and rows [smem_rows, split) are read from L2.
        const int c4 = tid & 63, jg = tid >> 6;                   // float4 c4 of both column halves; 8 j-groups
        const float4* ms = reinterpret_cast<const float4*>(rg.stage0 + mem_off);
        const float* mp = p.memory + (long)b * T * kEnc + c4 * 4;
        const int clen = p.infer ? len : T;
        const int split = p.infer ? staged_rows(len, len <= p.t4max ? 4 : 3) : staged_rows(T, p.nstages);
        float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;     // columns 4 c4 + [0, 4) and 256 + 4 c4 + [0, 4)
        auto fma4 = [](float4& acc, float a, const float4 m) {
          acc.x = fmaf(a, m.x, acc.x); acc.y = fmaf(a, m.y, acc.y); acc.z = fmaf(a, m.z, acc.z); acc.w = fmaf(a, m.w, acc.w);
        };
        int j = jg;
#pragma unroll 2
        for (; j < min(split, smem_rows); j += 8) {
          const float a = s_e[j];
          fma4(acc0, a, ms[j * (kEnc / 4) + c4]);
          fma4(acc1, a, ms[j * (kEnc / 4) + kEnc / 8 + c4]);
        }
        for (; j < split; j += 8) {                               // not staged
          const float a = s_e[j];
          fma4(acc0, a, __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc)));
          fma4(acc1, a, __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc + kEnc / 2)));
        }
        for (j = split + jg; j < clen; j += 8) {
          const float a = s_e[j];
          fma4(acc0, a, __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc)));
          fma4(acc1, a, __ldg(reinterpret_cast<const float4*>(mp + (long)j * kEnc + kEnc / 2)));
        }
        __syncthreads();                                          // everyone is done reading the staged rows
        float* scr = reinterpret_cast<float*>(rg.stage0);         // [8][512] partial sums
        *reinterpret_cast<float4*>(scr + jg * kEnc + c4 * 4) = acc0;
        *reinterpret_cast<float4*>(scr + jg * kEnc + kEnc / 2 + c4 * 4) = acc1;
        __syncthreads();
        if (tid < kEnc / 2) {
          const int col = tid * 2;
          float v0 = 0.f, v1 = 0.f;
#pragma unroll
          for (int g = 0; g < 8; ++g) { v0 += scr[g * kEnc + col]; v1 += scr[g * kEnc + col + 1]; }
          store_split2(p.ctx_img, b, col, v0, v1);
          if (p.st.ga)
            *reinterpret_cast<float2*>(p.st.ctx + ((long)(t + 1) * p.Btot + p.b0 + b) * kEnc + col) = make_float2(v0, v1);
        }
      }
      T2_PROF(19);
    }
    T2_PROF(5);
    grid_barrier(ctrl, bar_target);                                                             // B3: ctx_t complete
    T2_PROF(6);
    // ======== E2: ctx_t -> dec gates (rest), next att gates, projection (part); epilogue -> dh_t
    {
      // an upper CTA adds its partner's Ed sums (B3 ordered their stores) to its attention gate columns, while the
      // producer warp already issues E2's copies; warpgroup 1 adds E2's sums to those columns after this named barrier
      if (upper && warp > 0) {
        const float* part = p.part + (size_t)(cta - kAttCta0) * kRows * 32;
        for (int i = tid - 32; i < kRows * 32; i += kThreads - 32)
          s_acc[(i >> 5) * kAccPitch + kColA + (i & 31)] += __ldcg(part + i);
        asm volatile("bar.sync 1, %0;" ::"r"(kThreads - 32) : "memory");
      }
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
              // model.py:443; forced: the row's step count decides, its gate plays no part; limited: its gate or its own
              // step limit, whichever comes first
              if (!done && (kForced ? t + 1 == min(max(p.forced_lengths[row], 1), p.cap)
                                    : (sigmoid_exact(v) > p.gate_threshold ||
                                       (kLimited && p.max_steps && t + 1 == min(max(p.max_steps[row], 1), p.cap))))) {
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
      // The attention CTA is idle until x2 arrives and its ring is empty (E3 armed no next event): it computes the
      // location term of step t+1 from this step's attention weights, every round, into row b's block of p.pa.  A resumed
      // chunk reads it from there.  Its ah signal of step t+1 orders these stores before it copies the tile.
      if (!kForced && pa_pre && att_cta && t + 1 < p.cap)
        for (int r0 = 0; r0 < att_rounds; ++r0)
          att_pa_round(r0, pa_row + r0 * kAttRound, pa_p, min(T - r0 * kAttRound, kAttRound));
      T2_PROF(20);
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
      if (upper) {
        p.rs_att[((size_t)(cta - kAttCta0) * 2 + 0) * tpp + i] = s_pad0[i];
        p.rs_att[((size_t)(cta - kAttCta0) * 2 + 1) * tpp + i] = s_pad1[i];
      }
    }
    if (!is_lo) *rs_cell() = make_float4(c_att[0], c_att[1], c_dec[0], c_dec[1]);
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
// 0-93 at 4 stages and 0-57 at 3 for the attention context (fewer beside a precomputed pa tile); later rows are read
// from L2.
static int persistent_stages(int T) {
  int want = 4;
  const char* e = getenv("T2_STAGES");
  if (e && atoi(e) >= 3 && atoi(e) <= kMaxStages) want = atoi(e);
  while (want > 3 && persistent_smem_bytes(T, want) > kSmemLimit) --want;
  return want;
}

// the next step's location term of 64 rows (KParams::pa); none where no ring depth holds its tile
__host__ __device__ static size_t pa_buffer_floats(int T) { return pa_tile_fits(T, kMaxStages) ? (size_t)kRows * pa_tile_bytes(T) / 4 : 0; }
// whether a launch computes pa during the x2 wait (INFER, and the tile fits the ring it runs with)
static bool pa_precomputed(int T, bool infer) { return infer && pa_tile_fits(T, persistent_stages(T)); }

// ---------------------------------------------------------------------------------------------
// device state of the 64-row slices.  A slice buffer is the processed memory of all B rows (B, T_enc, 128), indexed by
// absolute row, then n_blocks slice blocks of one size: block i sits at blocks + i * stride.  t2_decoder_run has one block,
// which its consecutive 64-row launches reuse; a stream has one per slice, and those blocks also carry the state a launch
// saves at its end and restores at its start.
// ---------------------------------------------------------------------------------------------
constexpr size_t kSliceAlign = 1024;   // every region of a block, and the stride
struct SliceState {
  // every launch; a whole run zeroes the regions before pa with one memset
  DecoderCtrl* ctrl;                   // counters zeroed before every launch; a stream's stop latch is carried in `done`
  uint8_t *x2, *ah, *ctx, *dh, *x1;    // activation images of 4, 16, 8, 16 and 4 K chunks
  float* q;                            // (64, 128)
  float* pa;                           // location term of the next step (KParams::pa), pa_buffer_floats(T)
  float* part;                         // KParams::part
  // saved on-chip state (KParams::rs_*; streams only)
  float* acc; float* cell; float* att; int32_t* done;
};
__host__ __device__ static void slice_block_layout(Carve& c, int T, bool saved, SliceState* s) {
  s->ctrl = c.take<DecoderCtrl>(1, kSliceAlign);
  s->x2 = c.take<uint8_t>(4 * kXChunkBytes, kSliceAlign);
  s->ah = c.take<uint8_t>(16 * kXChunkBytes, kSliceAlign);
  s->ctx = c.take<uint8_t>(8 * kXChunkBytes, kSliceAlign);
  s->dh = c.take<uint8_t>(16 * kXChunkBytes, kSliceAlign);
  s->x1 = c.take<uint8_t>(4 * kXChunkBytes, kSliceAlign);
  s->q = c.take<float>((size_t)kRows * kAtt, kSliceAlign);
  s->pa = c.take<float>(pa_buffer_floats(T), kSliceAlign);
  s->part = c.take<float>((size_t)kAttCta0 * kRows * 32, kSliceAlign);   // KParams::part, written and read within a step
  s->acc = saved ? c.take<float>((size_t)kG * kRows * kAccPitch, kSliceAlign) : nullptr;
  s->cell = saved ? c.take<float>((size_t)kG * 4 * kRows * 4, kSliceAlign) : nullptr;
  s->att = saved ? c.take<float>((size_t)(kG - kAttCta0) * 2 * att_pad_len(T), kSliceAlign) : nullptr;
  s->done = saved ? c.take<int32_t>(kRows, kSliceAlign) : nullptr;
}

struct SliceBuffer {
  float* pm;                           // processed memory (B, T, 128)
  uint8_t* blocks; size_t stride;
  int T; bool saved;
  __host__ __device__ SliceState block(int i) const {
    Carve c(blocks + i * stride, 1);
    SliceState s;
    slice_block_layout(c, T, saved, &s);
    return s;
  }
};
__host__ __device__ static SliceBuffer slice_buffer_layout(Carve& c, int B, int T, int n_blocks, bool saved) {
  SliceBuffer b;
  b.T = T; b.saved = saved;
  b.pm = c.take<float>((size_t)B * T * kAtt, kSliceAlign);
  Carve one(nullptr, 1);
  SliceState s;
  slice_block_layout(one, T, saved, &s);
  b.stride = (one.off + kSliceAlign - 1) & ~(kSliceAlign - 1);
  b.blocks = c.take<uint8_t>((n_blocks - 1) * b.stride + one.off, kSliceAlign);
  return b;
}

// the persistent decoder's workspace: one slice block, then the teacher-forcing x2 images of every step (cap x 4 chunks)
static SliceBuffer persistent_ws_layout(Carve& c, int B, int T, int cap, uint8_t** teacher_img) {
  const SliceBuffer b = slice_buffer_layout(c, B, T, 1, false);
  *teacher_img = c.take<uint8_t>((size_t)cap * 4 * kXChunkBytes, kSliceAlign);
  return b;
}
size_t persistent_ws_bytes(int B, int T, int cap) {
  Carve c(nullptr, kDecoderWsAlign);
  uint8_t* teacher_img;
  persistent_ws_layout(c, B, T, cap, &teacher_img);
  return c.bytes();
}
DecoderCtrl* persistent_ws_ctrl(const T2DecoderArgs* a) {
  Carve c(a->ws, kDecoderWsAlign);
  uint8_t* teacher_img;
  return persistent_ws_layout(c, a->B, a->T_enc, a->n_steps_cap, &teacher_img).block(0).ctrl;
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
  // ---- per-CTA plans (host).  Consumers of an event are a contiguous run of [A | D | S].  E1 streams W_ih^d (D) on every
  // CTA and W_q (S) on the query CTAs; W_hh^a (A) of CTAs c and c + 64 is Ed of CTA c < 64 (its second consumer: the
  // partner's rows, stored to KParams::part) ----
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
    if (hq) set(1, 16, kColD, {32, 16}); else set(1, 16, kColD, {32});
    if (hp) set(2, 8, kColA, {32, 32, 16}); else set(2, 8, kColA, {32, 32});
    if (hp) set(3, 16, kColD, {32, 16}); else set(3, 16, kColD, {32});
    if (hx) set(4, 4, kColS, {16}); else { pl.ev[4].w_off = (uint32_t)off; }
    if (c < kAttCta0) set(kEd, 16, kColA, {32, 32}); else { pl.ev[kEd].w_off = (uint32_t)off; }
    for (int ev = 0; ev < kNumEvents; ++ev)
      if (pl.ev[ev].nrows != 0 && !event_plan_fits(pl.ev[ev])) return fail(T2_ERR_INVALID, "event plan does not fit the MMA warpgroups");
  }
  if (off >= (size_t)4 << 30) return fail(T2_ERR_INVALID, "W image too large");
  if (!pk->wimg) {
    pk->wimg_bytes = off + 1024;
    T2_CUDA(cudaMalloc((void**)&pk->wimg, pk->wimg_bytes));
    T2_CUDA(cudaMalloc((void**)&pk->plans, sizeof(CtaPlan) * kG));
    T2_CUDA(cudaMalloc((void**)&pk->wp_all, (size_t)kPCols * kdc * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_p, (size_t)kPCols * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_a, (size_t)kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->bias_d, (size_t)kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->rows, (size_t)5 * kG * 32 * 4));
    T2_CUDA(cudaMalloc((void**)&pk->weff, (size_t)kAtt * kChunkK * 4));
    T2_CUDA(cudaMalloc((void**)&pk->weff_img, (size_t)kWeffBytes));
  }
  fuse_location_kernel<<<kAtt, kChunkK, 0, s>>>(m->w[W_ATT_LOC_DENSE], m->w[W_ATT_LOC_CONV], pk->weff);
  T2_LAUNCH_CHECK();
  pack_rows_image_kernel<<<1, 256, 0, s>>>(pk->weff, kAtt, kChunkK, pk->weff_img);
  T2_LAUNCH_CHECK();
  T2_CUDA(cudaMemcpyAsync(pk->plans, plans.data(), sizeof(CtaPlan) * kG, cudaMemcpyHostToDevice, s));
  T2_CUDA(cudaStreamSynchronize(s));   // `plans` is a host temporary
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
  // ---- row tables: [0] LSTM gate rows, [1] q rows, [2] P rows, [3] x2 rows (S consumers: 8 real + 8 zero), [4] LSTM
  // gate rows of the partner CTA c + 64 (c < 64) ----
  std::vector<int32_t> rows((size_t)5 * kG * 32, -1);
  for (int c = 0; c < kG; ++c) {
    for (int col = 0; col < 32; ++col) rows[(0 * kG + c) * 32 + col] = (col & 3) * 1024 + c * 8 + (col >> 2);
    if (c < kAttCta0)
      for (int col = 0; col < 32; ++col) rows[(4 * kG + c) * 32 + col] = (col & 3) * 1024 + (c + kAttCta0) * 8 + (col >> 2);
    if (c >= kQCta0 && c < kQCta0 + kQCtas) for (int j = 0; j < 8; ++j) rows[(1 * kG + c) * 32 + j] = (c - kQCta0) * 8 + j;
    if (c >= kPCta0 && c < kPCta0 + kPCtas) for (int j = 0; j < 8; ++j) rows[(2 * kG + c) * 32 + j] = (c - kPCta0) * 8 + j;
    if (c >= kX2Cta0 && c < kX2Cta0 + kX2Ctas) for (int j = 0; j < 8; ++j) rows[(3 * kG + c) * 32 + j] = (c - kX2Cta0) * 8 + j;
  }
  T2_CUDA(cudaMemcpyAsync(pk->rows, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
  T2_CUDA(cudaStreamSynchronize(s));
  const int32_t* r_lstm = pk->rows; const int32_t* r_q = pk->rows + kG * 32;
  const int32_t* r_p = pk->rows + 2 * kG * 32; const int32_t* r_x2 = pk->rows + 3 * kG * 32;
  const int32_t* r_partner = pk->rows + 4 * kG * 32;
  // consumers [cons, cons + ncons) of one matrix, consumer cons + z with row table rt + z * tab_stride
  auto pack = [&](const float* src, int ld, int kcol0, int chunks, const int32_t* rt, int ev, int cons, int ncons = 1,
                  int tab_stride = 0) -> int {
    pack_consumer_kernel<<<dim3(chunks, kG, ncons), 256, 0, s>>>(src, ld, kcol0, rt, tab_stride, pk->plans, ev, cons, pk->wimg);
    T2_LAUNCH_CHECK();
    return T2_OK;
  };
  T2_TRY(pack(m->w[W_ARNN_WIH], kPre + kEnc, 0, 4, r_lstm, 0, 0));            // E0: att <- x2
  T2_TRY(pack(m->w[W_DRNN_WIH], kdc, 0, 16, r_lstm, 1, 0));                   // E1: dec <- ah
  T2_TRY(pack(m->w[W_ATT_QUERY], kARnn, 0, 16, r_q, 1, 1));                   //     q <- ah
  T2_TRY(pack(m->w[W_ARNN_WHH], kARnn, 0, 16, r_lstm, kEd, 0, 2,             // Ed: att' <- ah, partner's att' <- ah
              (int)(r_partner - r_lstm)));
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
  delete pk;
  m->pk = nullptr;
}

// processed_memory = memory_layer(memory) of batch rows [b0, b0 + nb) into their rows of pm (B, T, 128)  (model.py:288)
static int processed_memory(T2Model* m, const T2DecoderArgs* a, int b0, int nb, float* pm, cudaStream_t s) {
  GemmArgs g;
  g.seg[0] = {a->memory + (size_t)b0 * a->T_enc * kEnc, kEnc, m->w[W_ATT_MEMORY], kEnc, kEnc};
  g.M = nb * a->T_enc; g.N = kAtt; g.C = pm + (size_t)b0 * a->T_enc * kAtt; g.ldc = kAtt;
  return gemm_f32(g, s);
}

// the parameters of the launch over batch rows [b0, b0 + 64) (or to B) whose state is block `blk` of `buf`: the whole loop
// [0, cap), no resume state
static void slice_params(T2Model* m, const T2DecoderArgs* a, const SliceBuffer& buf, const SliceState& blk, int b0,
                         KParams* pp) {
  PersistentPack* pk = (PersistentPack*)m->pk;
  KParams& p = *pp;
  const int T = a->T_enc, cap = a->n_steps_cap;
  memset(&p, 0, sizeof(p));
  p.plans = pk->plans; p.wimg = pk->wimg; p.bias_a = pk->bias_a; p.bias_d = pk->bias_d; p.bias_p = pk->bias_p;
  p.weff_img = pk->weff_img; p.w_v = m->w[W_ATT_V];
  p.memory = a->memory + (size_t)b0 * T * kEnc; p.pm = buf.pm + (size_t)b0 * T * kAtt;
  p.mem_len = a->memory_lengths ? a->memory_lengths + b0 : nullptr;
  p.prenet_keep = a->prenet_keep; p.att_keep = a->att_keep; p.dec_keep = a->dec_keep;
  p.x2_img = blk.x2; p.ah_img = blk.ah; p.ctx_img = blk.ctx; p.dh_img = blk.dh; p.x1_img = blk.x1; p.q = blk.q;
  p.part = blk.part;
  p.mel = a->mel + (size_t)b0 * cap * kMel; p.gate = a->gate + (size_t)b0 * cap; p.align = a->align + (size_t)b0 * cap * T;
  p.mel_lengths = a->mel_lengths + b0; p.n_steps = a->n_steps;
  p.ctrl = blk.ctrl;
  p.b0 = b0; p.Btot = a->B;
  p.B = a->B - b0 < kRows ? a->B - b0 : kRows; p.T = T; p.cap = cap; p.infer = a->mode == T2_MODE_INFER;
  p.training = a->training;
  p.pa = pa_precomputed(T, p.infer) ? blk.pa : nullptr;
  p.gate_threshold = a->gate_threshold; p.score_mask_value = a->score_mask_value;
  p.p_att = m->cfg.p_attention_dropout; p.p_dec = m->cfg.p_decoder_dropout; p.seed = a->seed;
  p.row_seeds = a->row_seeds;
  p.t_begin = 0; p.t_end = cap;
  if (a->forced_align) {              // no location term: the forced kernel neither computes nor reads pa
    p.forced_align = a->forced_align + (size_t)b0 * cap * T; p.forced_lengths = a->forced_lengths + b0;
    p.pa = nullptr;
  }
  if (decoder_has_limits(a)) {
    // a window wider than T_enc on either side masks nothing, so no window (window_front == 0) and overly wide ones run
    // as (T_enc, T_enc); this also keeps p + win_front inside int
    p.win_back = a->window_front == 0 || a->window_back > T ? T : a->window_back;
    p.win_front = a->window_front == 0 || a->window_front > T ? T : a->window_front;
    p.max_steps = a->max_steps ? a->max_steps + b0 : nullptr;
  }
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
  void (*kernel)(KParams) = p.forced_align      ? decoder_persistent_kernel<kModeForced>
                            : p.win_front > 0 ? decoder_persistent_kernel<kModeLimited>
                                              : decoder_persistent_kernel<kModeFree>;
  T2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(kG); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeCooperative; attr.val.cooperative = 1;   // co-residency of all 128 CTAs
  cfg.attrs = &attr; cfg.numAttrs = 1;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, kernel, p);
  if (le != cudaSuccess) return fail(T2_ERR_CUDA, "persistent decoder launch failed: %s", cudaGetErrorString(le));
  if (getenv("T2_VERBOSE")) fprintf(stderr, "[t2b200] persistent decoder: B=%d T_enc=%d cap=%d stages=%d smem=%zu steps=%d-%d\n",
                                    p.B, p.T, p.cap, p.nstages, smem, p.t_begin, p.t_end);
  g_launch_count++;
  return T2_OK;
}

int decoder_run_persistent(T2Model* m, const T2DecoderArgs* a, cudaStream_t s) {
  const int cap = a->n_steps_cap;
  const bool infer = a->mode == T2_MODE_INFER;
  DecoderStash st;
  if (a->stash) {
    if (infer) return fail(T2_ERR_INVALID, "the training stash needs T2_MODE_TEACHER");
    if (a->stash_bytes < decoder_stash_bytes(a->B, cap)) return fail(T2_ERR_WORKSPACE, "decoder stash too small");
    Carve c(a->stash);
    decoder_stash_layout(c, a->B, cap, &st);
    float* z[5] = {st.ca, st.ha, st.cd, st.hd, st.ctx};   // slot 0 of the recurrent states = the zero initial states
    for (int i = 0; i < 5; ++i)                          // (model.py:258-284)
      T2_CUDA(cudaMemsetAsync(z[i], 0, (size_t)a->B * (i < 4 ? kARnn : kEnc) * sizeof(float), s));
  }
  Carve c(a->ws, kDecoderWsAlign);
  uint8_t* teacher_img;
  const SliceBuffer buf = persistent_ws_layout(c, a->B, a->T_enc, cap, &teacher_img);
  const SliceState blk = buf.block(0);
  T2_CUDA(cudaMemsetAsync(a->n_steps, 0, sizeof(int32_t), s));
  T2_TRY(processed_memory(m, a, 0, a->B, buf.pm, s));
  // batch rows are independent: more than 64 rows run as consecutive launches of <= 64 rows on the one block
  for (int b0 = 0; b0 < a->B; b0 += kRows) {
    KParams p;
    slice_params(m, a, buf, blk, b0, &p);
    // counters, zero images and q (model.py:258-284): the block's regions before pa
    T2_CUDA(cudaMemsetAsync(blk.ctrl, 0, (uint8_t*)blk.pa - (uint8_t*)blk.ctrl, s));
    if (p.pa) T2_CUDA(cudaMemsetAsync(p.pa, 0, pa_buffer_floats(a->T_enc) * 4, s));   // zero attention weights -> pa = +0.0
    p.st = st;
    if (!infer) {
      // teacher forcing (model.py:396-405): the prenet outputs of all steps are known up front -> convert
      // them once into x2 operand images, the kernel then skips the prenet events and their two barriers
      rows_to_image_kernel<<<dim3(4, cap), 256, 0, s>>>(a->teacher_prenet + (size_t)b0 * kPre, kPre, p.B, kPre,
                                                        (long)a->B * kPre, teacher_img, (long)4 * kXChunkBytes);
      T2_LAUNCH_CHECK();
      p.teacher_x2_img = teacher_img;
    }
    T2_TRY(launch_persistent(p, s));
  }
  return T2_OK;
}

// ---------------------------------------------------------------------------------------------
// resumable stream (t2_decoder_stream_*): the caller's state buffer is a slice buffer with one block per 64-row slice,
// saved state included
// ---------------------------------------------------------------------------------------------
__host__ __device__ static SliceBuffer stream_state_layout(Carve& c, int B, int T) {
  return slice_buffer_layout(c, B, T, (B + kRows - 1) / kRows, true);
}
static SliceBuffer stream_state(void* state, int B, int T) { Carve c(state, kSliceAlign); return stream_state_layout(c, B, T); }

size_t persistent_stream_state_bytes(int B, int T) { Carve c(nullptr, kSliceAlign); stream_state_layout(c, B, T); return c.bytes(); }

int persistent_stream_begin(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, cudaStream_t s) {
  T2_CUDA(cudaMemsetAsync(state, 0, persistent_stream_state_bytes(a->B, a->T_enc), s));   // model.py:258-284
  T2_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * ((a->B + kRows - 1) / kRows), s));
  T2_CUDA(cudaMemsetAsync(a->mel_lengths, 0xff, sizeof(int32_t) * a->B, s));                // -1: still live
  T2_CUDA(cudaMemsetAsync(a->n_steps, 0, sizeof(int32_t), s));
  return processed_memory(m, a, 0, a->B, stream_state(state, a->B, a->T_enc).pm, s);
}

int persistent_stream_run(T2Model* m, const T2DecoderArgs* a, void* state, int32_t* status, int n, const int32_t* status_host,
                          const int32_t* row_step0, cudaStream_t s) {
  const SliceBuffer buf = stream_state(state, a->B, a->T_enc);
  for (int b0 = 0, si = 0; b0 < a->B; b0 += kRows, ++si) {
    const int t0 = status_host ? status_host[2 * si] : 0;
    if ((status_host && status_host[2 * si + 1]) || t0 >= a->n_steps_cap) continue;    // this slice has stopped
    const SliceState blk = buf.block(si);
    T2_CUDA(cudaMemsetAsync(blk.ctrl, 0, sizeof(DecoderCtrl), s));   // everything else is zeroed by begin / admit
    KParams p;
    slice_params(m, a, buf, blk, b0, &p);                            // pa: left by the previous chunk
    p.t_begin = t0;
    p.t_end = n < a->n_steps_cap - t0 ? t0 + n : a->n_steps_cap;
    p.rs_acc = blk.acc; p.rs_cell = blk.cell; p.rs_att = blk.att; p.rs_done = blk.done; p.rs_status = status + 2 * si;
    p.row_step0 = row_step0;
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
  const int lr = blockIdx.x, row = blockIdx.y * kRows + lr, tid = threadIdx.x;
  if (row >= B || !((mask.w[row >> 6] >> (row & 63)) & 1ull)) return;
  Carve c(state, kSliceAlign);
  const SliceState sl = stream_state_layout(c, B, T).block(blockIdx.y);
  const int tpp = att_pad_len(T);
  for (int i = tid; i < kG * kAccPitch; i += 256)                  // its accumulator row in every CTA's tile
    sl.acc[((size_t)(i / kAccPitch) * kRows + lr) * kAccPitch + i % kAccPitch] = 0.f;
  for (int i = tid; i < kG * 4; i += 256)                          // its cell states: (CTA, column group)
    reinterpret_cast<float4*>(sl.cell)[(size_t)i * kRows + lr] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = tid; i < 2 * tpp; i += 256)                         // previous | cumulative weights of its attention CTA
    sl.att[(size_t)lr * 2 * tpp + i] = 0.f;
  const struct { uint8_t* img; int chunks; } imgs[5] = {{sl.x2, 4}, {sl.ah, 16}, {sl.ctx, 8}, {sl.dh, 16}, {sl.x1, 4}};
  for (const auto& im : imgs)
    for (int i = tid; i < im.chunks * 2 * (kChunkK / 2); i += 256) {   // its row in both planes of every chunk of an image
      const int chunk = i / kChunkK, plane = (i / (kChunkK / 2)) & 1, k = (i % (kChunkK / 2)) * 2;
      __half* pl = reinterpret_cast<__half*>(im.img + (size_t)chunk * kXChunkBytes) + plane * kRows * kChunkK;
      *reinterpret_cast<uint32_t*>(pl + img_elem_offset(lr, k)) = 0u;
    }
  for (int i = tid; i < kAtt; i += 256) sl.q[lr * kAtt + i] = 0.f;
  const size_t pa_row = pa_buffer_floats(T) / kRows;                // its pa tile (zero weights -> zero location term)
  for (size_t i = tid; i < pa_row; i += 256) sl.pa[lr * pa_row + i] = 0.f;
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
  // processed memory of the listed rows: one GEMM per run of consecutive rows (rows are ascending)
  float* pm = stream_state(state, a->B, a->T_enc).pm;
  for (int i = 0; i < n_rows;) {
    int j = i + 1;
    while (j < n_rows && rows[j] == rows[j - 1] + 1) ++j;
    T2_TRY(processed_memory(m, a, rows[i], j - i, pm, s));
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

}  // namespace t2
