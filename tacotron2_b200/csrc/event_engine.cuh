// The streaming "event" engine of the persistent decoder (decoder_persistent.cu), whose consumer plans, operand images
// and stage format the training backward's skinny GEMMs (decoder_backward.cu) share; those run their own ring, whose
// stages carry the activation chunks of two 64-row slices.  A CTA of 512 threads streams K chunks of a split-fp16 activation image [X_hi | X_lo] together
// with its weight rows through a shared-memory ring (bulk async copies issued by thread 0), and MMA warpgroups 1-3 each
// multiply one consumer's [W_hi; W_lo] rows with both activation planes and add the product to an fp32 accumulator tile
// in shared memory.
#pragma once
#include "decoder.h"
#include "umma.cuh"

namespace t2 {

constexpr int kThreads = 512;          // warp 0: bulk-copy producer; warpgroups 1-3: one consumer each
constexpr int kStages = 4;             // ring stages of the backward GEMMs
constexpr int kRows = 64;             // batch rows per launch (zero padded)
constexpr int kXChunkBytes = 2 * kRows * kChunkK * 2;    // [hi 64 rows | lo 64 rows] x 64 k fp16 = 16 KiB
constexpr int kHiCols = 80;                               // max weight rows of one event (hi)
constexpr int kAccPitch = 84;                             // floats per accumulator row (80 + 4: fewer bank conflicts)
constexpr int kAccBytes = kRows * kAccPitch * 4;
constexpr int kMmaWgs = 3;                                // warpgroups 1-3 issue the MMAs of an event (one piece each)
constexpr int kWStageMax = 2 * kHiCols * kChunkK * 2;    // hi + lo planes of up to 80 weight rows = 20 KiB
constexpr int kStageBytes = kXChunkBytes + kWStageMax;   // 36 KiB
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
// warpgroup 1 + c takes consumer c (n = 16 or 32 rows) as ONE wgmma B operand of N = 2 n rows [W_hi; W_lo] and multiplies
// it with A = X_hi and A = X_lo: two wgmma per 16-wide K step, each reading its activation plane and the consumer's rows
// once (instead of four with separate hi / lo B operands, each re-reading an A plane).  N stays <= 64 (32 accumulator
// registers): the decoder runs at the 128-register limit of 512 threads, and a wider accumulator spills.  Every consumer
// width is another copy of the chunk loop, and the decoder kernel runs its code once per step, so each width costs
// instruction-cache misses: the engine has exactly the two the plans need.
inline bool event_plan_fits(const EventPlan& ep) {
  if (ep.ncons < 1 || ep.ncons > kMmaWgs) return false;
  for (int c = 0; c < ep.ncons; ++c)
    if (ep.n[c] != 16 && ep.n[c] != 32) return false;
  return true;
}
// `rows` output rows of one matrix as consumers that fit the warpgroups: 32, 32, rest (rows <= 80, a multiple of 16)
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

// The chunk loop of one MMA warpgroup's consumer, shared by the decoder's events (NSL = 1) and the training backward's
// skinny GEMMs (NSL = 1 or 2 activation slices per stage): for each of `chunks` stages, D_s (64 x 2n) += X_s,hi . B^T +
// X_s,lo . B^T for every slice s, where X_s is the activation chunk at stage offset s x kXChunkBytes and B is the consumer's
// 2n weight-image rows [W_hi; W_lo] from row w_row0 of the weights at stage offset w_base.  Every slice sees its MMAs in
// the order of a one-slice event.  Each chunk's stage is released as soon as its MMAs are done: keeping a commit group in
// flight across chunks would hold every stage one chunk longer, i.e. make the ring one stage shallower for the producer,
// and the stream waits on L2 latency rather than on the tensor core (measured slower).
template <int N, int NSL>
__device__ __forceinline__ void event_mma(uint8_t* stage0, uint32_t stage_bytes, uint32_t w_base, uint32_t ns, uint64_t* full,
                                          uint64_t* empty, uint32_t& c_stage, uint32_t& c_phase, int chunks, uint32_t w_row0,
                                          DecoderCtrl* ctrl, float (&d)[NSL][N / 2]) {
  const bool leader = (threadIdx.x & 127) == 0;
  for (int i = 0; i < chunks; ++i) {
    mbar_wait(&full[c_stage], c_phase, ctrl, 201);
    const uint32_t xs = ptx::smem_u32(stage0 + c_stage * stage_bytes);
    const uint32_t ws = xs + w_base + w_row0 * 128;
#pragma unroll
    for (int s = 0; s < NSL; ++s) ptx::wg_fence_regs<N / 2>(d[s]);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < kChunkK / 16; ++kk) {
      const uint64_t b = ptx::make_sw128_desc(ws + kk * 32);
#pragma unroll
      for (int s = 0; s < NSL; ++s) {
        const uint32_t x = xs + s * kXChunkBytes;
        ptx::wgmma_f16<N>(d[s], ptx::make_sw128_desc(x + kk * 32), b);                  // X_hi
        ptx::wgmma_f16<N>(d[s], ptx::make_sw128_desc(x + kRows * 128 + kk * 32), b);    // X_lo
      }
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
#pragma unroll
    for (int s = 0; s < NSL; ++s) ptx::wg_fence_regs<N / 2>(d[s]);
    if (leader) ptx::mbar_arrive(&empty[c_stage]);
    if (++c_stage == ns) { c_stage = 0; c_phase ^= 1; }
  }
}

// One MMA warpgroup's consumer of an event: D (64 x 2n) = X_hi . B^T + X_lo . B^T over all `chunks` stages of the ring
// (event_mma); then the sum of both column halves of D is added to the accumulator tile from column acol, or, with out,
// stored to out (64 x n fp32, row-major) for another CTA to add to its tile.
template <int N>
__device__ __forceinline__ void event_wg(Ring& rg, int chunks, uint32_t w_row0, float* s_acc, int acol, DecoderCtrl* ctrl,
                                         float* out) {
  float d[1][N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[0][i] = 0.f;
  event_mma<N, 1>(rg.stage0, kStageBytes, kXChunkBytes, rg.ns, rg.full, rg.empty, rg.c_stage, rg.c_phase, chunks, w_row0, ctrl, d);
  const int wt = threadIdx.x & 127;
#pragma unroll
  for (int j = 0; j < N / 4; ++j) {    // registers [0, N/4) hold the W_hi columns, [N/4, N/2) the W_lo ones
    const float v = d[0][j] + d[0][N / 4 + j];
    if (out) out[ptx::wg_frag_row(j, wt) * (N / 2) + ptx::wg_frag_col(j, wt)] = v;
    else s_acc[ptx::wg_frag_row(j, wt) * kAccPitch + acol + ptx::wg_frag_col(j, wt)] += v;
  }
}

// Streams `chunks` K-chunks of the activation image x_img plus this CTA's weight rows through the ring;
// warpgroups 1-3 issue the MMAs (one consumer each) and add their products to the accumulator tile s_acc.  Called by all threads;
// returns after the accumulators are complete.  Every MMA accumulates (the epilogues zero what they consume).
// The plan's consumers have 32 or 16 rows (event_plan_fits).  out_last (or null): the last consumer's sums go there
// (event_wg) instead of into s_acc.
__device__ __forceinline__ void run_event(Ring& rg, const EventPlan& ep, const uint8_t* x_img,
                                          const uint8_t* w_img, int chunks, float* s_acc,
                                          DecoderCtrl* ctrl, const EventPlan* next,
                                          const unsigned int* ready = nullptr, unsigned int ready_target = 0,
                                          float* out_last = nullptr) {
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
      float* out = c == ep.ncons - 1 ? out_last : nullptr;
      if (ep.n[c] == 32) event_wg<64>(rg, chunks, w_row0, s_acc, acol, ctrl, out);
      else event_wg<32>(rg, chunks, w_row0, s_acc, acol, ctrl, out);
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

}  // namespace t2
