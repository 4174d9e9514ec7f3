// General fp32-grade GEMM of the training path on the tensor cores (wgmma, split fp16); every dense product of the
// training path that is not a time-batched LSTM weight gradient (wgrad_tc.cu) or a conv input gradient (conv_tc.cu):
//
//     C (M x N, row-major, ldc) = op(A) . op(B) + beta * C        ta: A is stored (K x M), tb: B is stored (N x K)
//
// fp32 operands are converted ON THE FLY: a CTA (256 threads) loads a 128 x 64 tile of op(A) and a 128 x 64 tile of
// op(B)^T from global memory (coalesced along whichever dimension is contiguous), multiplies every row of op(A) / column
// of op(B) by a power of two derived from its largest magnitude over K (a pre-pass; gradients span many orders of
// magnitude, fp16 does not), splits x = hi + lo into two fp16 planes and writes them as K-major SWIZZLE_128B operand
// images into shared memory (double buffered).  Two warpgroups issue hi.hi + lo.hi + hi.lo per 16-wide K step, each into
// 64 x 128 fp32 register accumulators.  Long accumulation chains on the tensor cores lose accuracy (DESIGN.md section 4),
// so every K chunk is its own chain (hi.hi and the cross terms in separate accumulators), added to fp32 running sums
// (64 per thread) once the chunk's MMAs completed.  Small-tile /
// large-K shapes (the time-batched weight gradients: K = T x B = 51,200) are split along K over CTAs; the partial tiles
// are added in a fixed order by a reduce kernel (bit-reproducible).
#include <stdlib.h>
#include <string.h>

#include "gemm_tc.h"
#include "umma.cuh"

namespace t2 {

namespace {

constexpr int kBM = 128, kBN = 128, kBK = 64;
constexpr int kThreadsG = 256;
constexpr int kPlane = 128 * 128;                 // one fp16 plane of 128 rows x 64 k = 16 KiB
constexpr int kBufBytes = 4 * kPlane;             // [A hi | A lo | B hi | B lo]
constexpr int kTargetExp = 13;                    // scaled row / column maximum in [2^13, 2^14)

// ---- pre-pass: largest magnitude of every row of op(A) / column of op(B) over K (as raw float bits, atomicMax) ------
// inner (K) contiguous: one warp per outer index.  blockIdx.z: batch entry at element stride s_batch, with its own
// n_outer maxima in out; outer_of (device, per entry, or nullptr): the entry's outer indices past it are not read.
__global__ void absmax_inner_contig_kernel(const float* __restrict__ X, long s_outer, int n_outer, int n_inner,
                                           unsigned int* __restrict__ out, long s_batch, const int* __restrict__ outer_of) {
  const int o = blockIdx.x * blockDim.y + threadIdx.y;
  if (o >= (outer_of ? min(n_outer, outer_of[blockIdx.z]) : n_outer)) return;
  const long per = (n_inner + gridDim.y - 1) / gridDim.y;
  const long i0 = blockIdx.y * per, i1 = i0 + per < n_inner ? i0 + per : n_inner;
  float mx = 0.f;
  const float* r = X + blockIdx.z * s_batch + (long)o * s_outer;
  out += (long)blockIdx.z * n_outer;
  for (long i = i0 + threadIdx.x; i < i1; i += 32) mx = fmaxf(mx, fabsf(r[i]));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  if (threadIdx.x == 0 && mx > 0.f) atomicMax(out + o, __float_as_uint(mx));
}
// outer contiguous: thread x = outer index, y strides over the K rows
__global__ void absmax_outer_contig_kernel(const float* __restrict__ X, long s_inner, int n_outer, int n_inner,
                                           unsigned int* __restrict__ out) {
  __shared__ float red[8][33];
  const int o = blockIdx.x * 32 + threadIdx.x;
  const long per = (n_inner + gridDim.y - 1) / gridDim.y;
  const long i0 = blockIdx.y * per, i1 = i0 + per < n_inner ? i0 + per : n_inner;
  float mx = 0.f;
  if (o < n_outer)
    for (long i = i0 + threadIdx.y; i < i1; i += 8) mx = fmaxf(mx, fabsf(X[i * s_inner + o]));
  red[threadIdx.y][threadIdx.x] = mx;
  __syncthreads();
  if (threadIdx.y == 0 && o < n_outer) {
    for (int y = 1; y < 8; ++y) mx = fmaxf(mx, red[y][threadIdx.x]);
    if (mx > 0.f) atomicMax(out + o, __float_as_uint(mx));
  }
}

// power of two s with max * s in [2^kTargetExp, 2^(kTargetExp+1)); non-finite or zero maxima -> 1
__device__ __forceinline__ float scale_of(unsigned int bits) {
  const int e = (int)((bits >> 23) & 0xffu);
  if (e == 0 || e == 255) return 1.f;
  int se = 127 + kTargetExp - (e - 127);          // biased exponent of the scale
  se = se < 1 ? 1 : (se > 254 ? 254 : se);
  return __uint_as_float((unsigned int)se << 23);
}

struct GemmP {
  const float* A; const float* B; float* C; float* part;     // part != nullptr: write partial tiles (split K)
  const unsigned int* amax; const unsigned int* bmax;
  long lda, ldb, ldc, sA, sB, sC;                              // leading dimensions, batch strides (elements)
  int M, N, K, ta, tb, splits, chunks_per_split, batch;
  float beta;
  const int* entry_rows; int sms;                              // ragged entries (GemmTc::entry_rows), planned for sms
};

// The split rule: small-tile / large-K problems are split along K so that they fill one wave of CTAs (1 CTA / SM:
// 161 KiB of shared memory).  Scratch: [amax (M)][bmax (N)][partial tiles of the K splits].  The ragged kernel evaluates
// it on the device for each entry's own row count.
struct Plan { int ntm, ntn, splits, cps; long tiles; size_t off_part, bytes; };
__host__ __device__ Plan plan(int M, int N, int K, int batch, int sms) {
  Plan p;
  p.ntm = (M + kBM - 1) / kBM; p.ntn = (N + kBN - 1) / kBN;
  const int nchunks = (K + kBK - 1) / kBK;
  p.tiles = (long)p.ntm * p.ntn * batch;
  int splits = 1;
  if (p.tiles * 5 < sms * 4 && nchunks >= 8) {
    splits = p.tiles <= sms / 2 ? (int)(sms / p.tiles) : 2;
    if (splits > nchunks / 4) splits = nchunks / 4;
    if (splits < 1) splits = 1;
  }
  p.cps = (nchunks + splits - 1) / splits;
  p.splits = (nchunks + p.cps - 1) / p.cps;
  p.off_part = (((size_t)M + N) * 4 + 255) & ~(size_t)255;
  p.bytes = p.off_part + (p.splits > 1 ? (size_t)p.tiles * p.splits * kBM * kBN * 4 : 0);
  return p;
}

// ---- operand tiles: global fp32 -> registers -> (transposing stage) -> split-fp16 SWIZZLE_128B planes -----------------
// Every thread owns 4 groups of 8 consecutive elements of the 128 x 64 tile.  `kc`: the K dimension is contiguous in
// memory (element (r, k) at X[r * ld + k]): group = 8 consecutive k of one row.  Otherwise the row dimension is
// contiguous (element at X[k * ld + r]): group = 8 consecutive rows at one k, and the tile is transposed through a
// padded fp32 staging tile in shared memory (conflict-free both ways) instead of scattered 2-byte stores.
constexpr int kStagePitch = 132;                                   // floats per k-row of the staging tile (128 + 4)
constexpr int kStageBytesG = kBK * kStagePitch * 4;                // 33,792 B

__device__ __forceinline__ void load8(const float* __restrict__ src, bool vec, int n_valid, float (&v)[8]) {
  if (vec) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (e < n_valid) ? __ldg(src + e) : 0.f;
  }
}
// issue the global loads of one operand tile (no dependent instruction: all 4 x 32 B per thread are in flight together)
__device__ __forceinline__ void tile_fetch(const float* __restrict__ X, long ld, bool kc, int r0, int k0, int R, int K,
                                           float (&v)[4][8]) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int item = tid + q * kThreadsG;
    if (kc) {
      const int r = item >> 3, g8 = item & 7, row = r0 + r, k = k0 + g8 * 8;
      if (row < R && k < K) {
        const float* src = X + (long)row * ld + k;
        load8(src, k + 8 <= K && ((reinterpret_cast<uintptr_t>(src) & 15) == 0), K - k, v[q]);
        continue;
      }
    } else {
      const int kk = item >> 4, mg = item & 15, k = k0 + kk, row = r0 + mg * 8;
      if (k < K && row < R) {
        const float* src = X + (long)k * ld + row;
        load8(src, row + 8 <= R && ((reinterpret_cast<uintptr_t>(src) & 15) == 0), R - row, v[q]);
        continue;
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) v[q][e] = 0.f;
  }
}
// registers -> scaled split-fp16 planes.  The transposing path needs two CTA-wide barriers (stage written / stage read).
__device__ __forceinline__ void tile_store(const float (&v)[4][8], bool kc, int r0, int R, const unsigned int* __restrict__ rmax,
                                           float* __restrict__ stage, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int tid = threadIdx.x;
  if (kc) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int item = tid + q * kThreadsG, r = item >> 3, g8 = item & 7;
      const float sc = (r0 + r < R) ? scale_of(rmax[r0 + r]) : 1.f;
      __align__(16) __half hh[8];
      __align__(16) __half ll[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) split_fp16(v[q][e] * sc, hh[e], ll[e]);
      const uint32_t off = (uint32_t)((r >> 3) * 512 + (r & 7) * 64 + ((g8 ^ (r & 7)) * 8));
      *reinterpret_cast<uint4*>(hi + off) = *reinterpret_cast<const uint4*>(hh);
      *reinterpret_cast<uint4*>(lo + off) = *reinterpret_cast<const uint4*>(ll);
    }
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int item = tid + q * kThreadsG, kk = item >> 4, mg = item & 15;
      float* d = stage + kk * kStagePitch + mg * 8;
      *reinterpret_cast<float4*>(d) = make_float4(v[q][0], v[q][1], v[q][2], v[q][3]);
      *reinterpret_cast<float4*>(d + 4) = make_float4(v[q][4], v[q][5], v[q][6], v[q][7]);
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int item = tid + q * kThreadsG, r = item & 127, g8 = item >> 7;       // lanes along the rows: conflict-free reads
      const float sc = (r0 + r < R) ? scale_of(rmax[r0 + r]) : 1.f;
      __align__(16) __half hh[8];
      __align__(16) __half ll[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) split_fp16(stage[(g8 * 8 + e) * kStagePitch + r] * sc, hh[e], ll[e]);
      const uint32_t off = (uint32_t)((r >> 3) * 512 + (r & 7) * 64 + ((g8 ^ (r & 7)) * 8));
      *reinterpret_cast<uint4*>(hi + off) = *reinterpret_cast<const uint4*>(hh);
      *reinterpret_cast<uint4*>(lo + off) = *reinterpret_cast<const uint4*>(ll);
    }
    __syncthreads();                        // the stage may be overwritten by the next operand
  }
}

// Shared memory: [2 operand buffers x 64 KiB][transposing stage 33 KiB]; the epilogue's output tile reuses the operand
// buffers.  Warpgroup w (threads 128 w ..) owns rows [64 w, 64 w + 64) of the tile: per K chunk it issues hi.hi into one
// register accumulator and the cross terms (lo.hi, hi.lo) into another (4 / 8 wgmma of 64 x 128 x 16), waits for them
// and adds both to its fp32 running sums -- one accumulation chain = ONE K chunk: the tensor core's accumulator update
// truncates, so the error grows with the chain length; 4 / 8 accumulations per chain keep the result at fp32 sgemm
// quality (~1e-7).  The operand buffers are double buffered, so one CTA-wide barrier per chunk orders the next chunk's
// stores after the MMAs that read the same buffer two chunks earlier.
constexpr int kSmemG = 2 * kBufBytes + kStageBytesG;

// Ragged entries: add split sp's partial tile, scaled back exactly as the epilogue does, to the entry's C, and restart
// the accumulators.  As splitk_reduce_kernel, a split plan sums from +0 in split order and an unsplit one stores the
// tile as it is.  Each thread reads back only what it wrote itself.
__device__ __forceinline__ void ragged_fold(const GemmP& p, float (&acc)[64], int batch, int M, int m0, int n0,
                                            const unsigned int* __restrict__ amax, int splits, int sp) {
  const int wg = threadIdx.x >> 7, wt = threadIdx.x & 127;
  float* Cb = p.C + (long)batch * p.sC;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int m = m0 + wg * 64 + ptx::wg_frag_row(i, wt), n = n0 + ptx::wg_frag_col(i, wt);
    if (m < M && n < p.N) {
      const float ia = 1.f / scale_of(amax[m]);
      const float v = __fmul_rn(acc[i], ia / scale_of(p.bmax[n]));
      float* dst = Cb + (long)m * p.ldc + n;
      *dst = splits == 1 ? v : __fadd_rn(sp == 0 ? 0.f : *dst, v);
    }
    acc[i] = 0.f;
  }
}

// kRagged (GemmTc::entry_rows): one CTA per (entry, tile) runs the entry's K splits one after the other and adds each
// split's scaled partial tile to C in the order splitk_reduce_kernel adds them, so every entry gets the bits of its own
// batch = 1 call.
template <bool kRagged>
__global__ void __launch_bounds__(kThreadsG, 1) gemm_tc_kernel(const GemmP p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  float* stage = reinterpret_cast<float*>(smem_raw + 2 * kBufBytes);
  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;
  const int bz = blockIdx.z, batch = kRagged ? bz : bz / p.splits, split = kRagged ? 0 : bz - batch * p.splits;
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const float* A = p.A + (long)batch * p.sA;
  const float* B = p.B + (long)batch * p.sB;
  const int nchunks = (p.K + kBK - 1) / kBK;
  int M = p.M, cps = p.chunks_per_split, splits = 1;
  const unsigned int* amax = p.amax;
  if constexpr (kRagged) {
    M = min(p.M, p.entry_rows[batch]);
    if (m0 >= M) return;                    // the whole CTA: past the entry's rows
    const Plan pl = plan(M, p.N, p.K, 1, p.sms);
    cps = pl.cps; splits = pl.splits;
    amax += (long)batch * p.M;
  }
  const int c0 = split * cps, c1 = kRagged ? nchunks : min(nchunks, c0 + cps);
  const bool a_kc = !p.ta, b_kc = p.tb != 0;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  int it = 0;
  for (int c = c0; c < c1; ++c, ++it) {
    if constexpr (kRagged) {
      if (c > 0 && c % cps == 0) ragged_fold(p, acc, batch, M, m0, n0, amax, splits, c / cps - 1);
    }
    uint8_t* sb = smem_raw + (it & 1) * kBufBytes;
    {
      float va[4][8], vb[4][8];
      tile_fetch(A, p.lda, a_kc, m0, c * kBK, M, p.K, va);         // both operands' loads in flight together
      tile_fetch(B, p.ldb, b_kc, n0, c * kBK, p.N, p.K, vb);
      tile_store(va, a_kc, m0, M, amax, stage, reinterpret_cast<__half*>(sb), reinterpret_cast<__half*>(sb + kPlane));
      tile_store(vb, b_kc, n0, p.N, p.bmax, stage, reinterpret_cast<__half*>(sb + 2 * kPlane), reinterpret_cast<__half*>(sb + 3 * kPlane));
    }
    ptx::fence_proxy_async();
    __syncthreads();
    const uint32_t a_hi = ptx::smem_u32(sb) + (uint32_t)wg * (64 * 128), a_lo = a_hi + kPlane;
    const uint32_t b_hi = ptx::smem_u32(sb) + 2 * kPlane, b_lo = b_hi + kPlane;
    float dh[64], dx[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { dh[i] = 0.f; dx[i] = 0.f; }
    ptx::wg_fence_regs<64>(dh);
    ptx::wg_fence_regs<64>(dx);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < kBK / 16; ++kk) {
      const uint64_t dah = ptx::make_sw128_desc(a_hi + kk * 32), dal = ptx::make_sw128_desc(a_lo + kk * 32);
      const uint64_t dbh = ptx::make_sw128_desc(b_hi + kk * 32), dbl = ptx::make_sw128_desc(b_lo + kk * 32);
      ptx::wgmma_f16<kBN>(dh, dah, dbh);
      ptx::wgmma_f16<kBN>(dx, dal, dbh);
      ptx::wgmma_f16<kBN>(dx, dah, dbl);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::wg_fence_regs<64>(dh);
    ptx::wg_fence_regs<64>(dx);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += dh[i] + dx[i];
  }
  if constexpr (kRagged) {
    ragged_fold(p, acc, batch, M, m0, n0, amax, splits, splits - 1);
    return;
  }
  __syncthreads();                          // every MMA is complete: the operand buffers become the output tile

  // ---- epilogue: undo the scales, transpose through shared memory, coalesced stores -----------------------------------
  float* tile = reinterpret_cast<float*>(smem_raw);                 // [128][kStagePitch]
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int r = wg * 64 + ptx::wg_frag_row(i, wt), col = ptx::wg_frag_col(i, wt);
    const int m = m0 + r, n = n0 + col;
    const float ia = (m < p.M) ? 1.f / scale_of(p.amax[m]) : 0.f;
    tile[r * kStagePitch + col] = acc[i] * (ia / scale_of(n < p.N ? p.bmax[n] : 0u));
  }
  __syncthreads();
  if (p.part) {                             // partial tile of this K split: contiguous 128 x 128
    float* dst = p.part + (((long)bz * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * (long)(kBM * kBN);
    for (int idx = tid; idx < kBM * (kBN / 4); idx += kThreadsG) {
      const int r = idx >> 5, c4 = idx & 31;
      *reinterpret_cast<float4*>(dst + r * kBN + c4 * 4) = *reinterpret_cast<const float4*>(tile + r * kStagePitch + c4 * 4);
    }
  } else {
    float* Cb = p.C + (long)batch * p.sC;
    const bool vec = (p.ldc & 3) == 0 && ((reinterpret_cast<uintptr_t>(Cb) & 15) == 0) && n0 + kBN <= p.N;
    if (vec) {
      for (int idx = tid; idx < kBM * (kBN / 4); idx += kThreadsG) {
        const int r = idx >> 5, c4 = idx & 31, m = m0 + r;
        if (m >= p.M) continue;
        float4 v = *reinterpret_cast<const float4*>(tile + r * kStagePitch + c4 * 4);
        float4* dst = reinterpret_cast<float4*>(Cb + (long)m * p.ldc + n0 + c4 * 4);
        if (p.beta != 0.f) {
          const float4 o = *dst;
          v.x = fmaf(p.beta, o.x, v.x); v.y = fmaf(p.beta, o.y, v.y); v.z = fmaf(p.beta, o.z, v.z); v.w = fmaf(p.beta, o.w, v.w);
        }
        *dst = v;
      }
    } else {
      for (int idx = tid; idx < kBM * kBN; idx += kThreadsG) {
        const int r = idx >> 7, cidx = idx & 127, m = m0 + r, n = n0 + cidx;
        if (m >= p.M || n >= p.N) continue;
        float v = tile[r * kStagePitch + cidx];
        float* dst = Cb + (long)m * p.ldc + n;
        if (p.beta != 0.f) v = fmaf(p.beta, *dst, v);
        *dst = v;
      }
    }
  }
}

// C = beta C + sum over the K splits of the partial tiles, fixed order
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int batch, int ntm, int ntn, int M, int N,
                                     float* __restrict__ C, long ldc, long sC, float beta) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long per_batch = (long)M * N;
  if (idx >= per_batch * batch) return;
  const int b = (int)(idx / per_batch);
  const long r = idx - (long)b * per_batch;
  const int m = (int)(r / N), n = (int)(r - (long)m * N);
  const int tm = m / kBM, tn = n / kBN;
  float s = 0.f;
  for (int sp = 0; sp < splits; ++sp) {
    const long bz = (long)b * splits + sp;
    s += part[((bz * ntm + tm) * ntn + tn) * (long)(kBM * kBN) + (long)(m - tm * kBM) * kBN + (n - tn * kBN)];
  }
  float* c = C + (long)b * sC + (long)m * ldc + n;
  *c = beta != 0.f ? fmaf(beta, *c, s) : s;
}

// column sums: out[c] = sum over rows of X[r * ld + c]  (the bias gradients; replaces ones-vector GEMMs).  Rows are cut
// in kColSplit segments summed in fp32, the segment sums are added in double in a fixed order.
constexpr int kColSplit = 64;                   // at most; few-row inputs use fewer (gridDim.y)
__global__ void __launch_bounds__(256) colsum_part_kernel(const float* __restrict__ X, long ld, long rows, int cols,
                                                          float* __restrict__ part) {
  __shared__ float red[8][33];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const long per = (rows + gridDim.y - 1) / gridDim.y;
  const long r0 = blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
  float sm = 0.f;
  if (c < cols)
    for (long r = r0 + rg; r < r1; r += 8) sm += X[r * ld + c];
  red[rg][cl] = sm;
  __syncthreads();
  if (rg == 0 && c < cols) {
    for (int i = 1; i < 8; ++i) sm += red[i][cl];
    part[(long)blockIdx.y * cols + c] = sm;
  }
}
__global__ void colsum_final_kernel(const float* __restrict__ part, int nsplit, int cols, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  double s = 0.0;
  for (int i = 0; i < nsplit; ++i) s += (double)part[(long)i * cols + c];
  out[c] = (float)s;
}

}  // namespace

// The split count never falls as the SM count grows, so the plan for a full GH100 (144 SMs) bounds every sm_90a device.
size_t gemm_tc_ws_bytes(int M, int N, int K, int batch) {
  return M > 0 && N > 0 && K > 0 ? plan(M, N, K, batch > 0 ? batch : 1, 144).bytes : 0;
}
// ragged entries: [amax (batch x M)][bmax (N)], no partial tiles
size_t gemm_tc_ragged_ws_bytes(int M, int N, int batch) {
  return M > 0 && N > 0 ? (((size_t)(batch > 0 ? batch : 1) * M + N) * 4 + 255) & ~(size_t)255 : 0;
}

// K splits of the maximum search: enough blocks to saturate HBM on the long-K operands (K up to 7.7 M rows)
static int absmax_k_splits(int K) {
  int ysp = K >= 4096 ? 32 : (K >= 512 ? 4 : 1);
  if (K >= (1 << 16)) { ysp = K >> 9; if (ysp > 1024) ysp = 1024; }
  return ysp;
}
static int launch_bmax(cudaStream_t s, const GemmTc& g, const float* B, int ysp, unsigned int* bmax) {
  if (g.tb) absmax_inner_contig_kernel<<<dim3((g.N + 7) / 8, ysp), dim3(32, 8), 0, s>>>(B, g.ldb, g.N, g.K, bmax, 0, nullptr);
  else absmax_outer_contig_kernel<<<dim3((g.N + 31) / 32, ysp), dim3(32, 8), 0, s>>>(B, g.ldb, g.N, g.K, bmax);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

static GemmP gemm_params(const GemmTc& g, int batch, unsigned int* amax, unsigned int* bmax) {
  GemmP p;
  memset(&p, 0, sizeof(p));
  p.A = g.A; p.B = g.B; p.C = g.C; p.amax = amax; p.bmax = bmax;
  p.lda = g.lda; p.ldb = g.ldb; p.ldc = g.ldc; p.sA = g.strideA; p.sB = g.strideB; p.sC = g.strideC;
  p.M = g.M; p.N = g.N; p.K = g.K; p.ta = g.ta ? 1 : 0; p.tb = g.tb ? 1 : 0; p.batch = batch; p.beta = g.beta;
  return p;
}

// Ragged entries (GemmTc::entry_rows): one pre-pass launch for the row maxima of every entry, one for the shared op(B),
// one GEMM launch whose CTAs past an entry's rows exit at once.
static int gemm_tc_ragged(int sm_count, cudaStream_t s, const GemmTc& g, int batch) {
  if (g.ta || g.strideB != 0 || g.beta != 0.f)
    return fail(T2_ERR_INVALID, "gemm_tc: ragged entries need a K-contiguous op(A), one op(B) and beta = 0");
  const size_t need = gemm_tc_ragged_ws_bytes(g.M, g.N, batch);
  if (g.ws_bytes < need) return fail(T2_ERR_WORKSPACE, "gemm_tc: scratch of %zu bytes, %zu needed", g.ws_bytes, need);
  unsigned int* amax = (unsigned int*)g.ws;
  unsigned int* bmax = amax + (size_t)batch * g.M;
  T2_CUDA(cudaMemsetAsync(g.ws, 0, ((size_t)batch * g.M + g.N) * 4, s));
  const int ysp = absmax_k_splits(g.K);
  absmax_inner_contig_kernel<<<dim3((g.M + 7) / 8, ysp, batch), dim3(32, 8), 0, s>>>(g.A, g.lda, g.M, g.K, amax, g.strideA,
                                                                                    g.entry_rows);
  T2_LAUNCH_CHECK();
  T2_TRY(launch_bmax(s, g, g.B, ysp, bmax));
  GemmP p = gemm_params(g, batch, amax, bmax);
  p.entry_rows = g.entry_rows; p.sms = sm_count;
  const Plan pl = plan(g.M, g.N, g.K, 1, sm_count);
  T2_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemG));
  gemm_tc_kernel<true><<<dim3(pl.ntn, pl.ntm, batch), kThreadsG, kSmemG, s>>>(p);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int gemm_tc(int sm_count, cudaStream_t s, const GemmTc& g) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return fail(T2_ERR_INVALID, "gemm_tc: empty problem %d x %d x %d", g.M, g.N, g.K);
  const int batch = g.batch > 0 ? g.batch : 1;
  if (g.entry_rows) return gemm_tc_ragged(sm_count, s, g, batch);
  const Plan pl = plan(g.M, g.N, g.K, batch, sm_count);
  const int ntm = pl.ntm, ntn = pl.ntn, splits = pl.splits, cps = pl.cps;
  if (g.ws_bytes < pl.bytes) return fail(T2_ERR_WORKSPACE, "gemm_tc: scratch of %zu bytes, %zu needed", g.ws_bytes, pl.bytes);
  const size_t n_a = (size_t)g.M, n_b = (size_t)g.N;
  char* ws = (char*)g.ws;
  unsigned int* amax = (unsigned int*)ws;
  unsigned int* bmax = amax + n_a;
  // one scale per row of op(A) / column of op(B), shared by the batch entries (maximum over the batch)
  T2_CUDA(cudaMemsetAsync(ws, 0, (n_a + n_b) * 4, s));
  for (int b = 0; b < batch; ++b) {
    const float* A = g.A + (long)b * g.strideA;
    const float* B = g.B + (long)b * g.strideB;
    const int ysp = absmax_k_splits(g.K);
    if (!g.ta) absmax_inner_contig_kernel<<<dim3((g.M + 7) / 8, ysp), dim3(32, 8), 0, s>>>(A, g.lda, g.M, g.K, amax, 0, nullptr);
    else absmax_outer_contig_kernel<<<dim3((g.M + 31) / 32, ysp), dim3(32, 8), 0, s>>>(A, g.lda, g.M, g.K, amax);
    T2_LAUNCH_CHECK();
    T2_TRY(launch_bmax(s, g, B, ysp, bmax));
  }
  GemmP p = gemm_params(g, batch, amax, bmax);
  p.part = splits > 1 ? (float*)(ws + pl.off_part) : nullptr;
  p.splits = splits; p.chunks_per_split = cps;
  const size_t smem = (size_t)kSmemG;
  T2_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  gemm_tc_kernel<false><<<dim3(ntn, ntm, batch * splits), kThreadsG, smem, s>>>(p);
  T2_LAUNCH_CHECK();
  if (splits > 1) {
    const long total = (long)g.M * g.N * batch;
    splitk_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(p.part, splits, batch, ntm, ntn, g.M, g.N, g.C, g.ldc,
                                                                        g.strideC, g.beta);
    T2_LAUNCH_CHECK();
  }
  return T2_OK;
}

int gemm_tc_rm(int sm_count, cudaStream_t s, void* ws, size_t ws_bytes, bool ta, bool tb, int M, int N, int K, const float* A,
               long lda, const float* B, long ldb, float* C, long ldc, float beta) {
  GemmTc g;
  g.ta = ta; g.tb = tb; g.M = M; g.N = N; g.K = K; g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc; g.beta = beta;
  g.ws = ws; g.ws_bytes = ws_bytes;
  return gemm_tc(sm_count, s, g);
}

static int colsum_splits(long rows) {
  const long nsplit = rows / 64;
  return nsplit < 1 ? 1 : (nsplit > kColSplit ? kColSplit : (int)nsplit);
}
size_t colsum_ws_bytes(long rows, int cols) { return (size_t)colsum_splits(rows) * cols * 4; }

int colsum_f32(cudaStream_t s, void* ws, size_t ws_bytes, const float* X, long ld, long rows, int cols, float* out) {
  if (rows <= 0 || cols <= 0) return fail(T2_ERR_INVALID, "colsum: empty input");
  const int nsplit = colsum_splits(rows);
  if (ws_bytes < colsum_ws_bytes(rows, cols)) return fail(T2_ERR_WORKSPACE, "colsum: scratch too small");
  colsum_part_kernel<<<dim3((cols + 31) / 32, nsplit), 256, 0, s>>>(X, ld, rows, cols, (float*)ws);
  T2_LAUNCH_CHECK();
  colsum_final_kernel<<<(cols + 255) / 256, 256, 0, s>>>((const float*)ws, nsplit, cols, out);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
