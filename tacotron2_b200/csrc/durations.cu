// Duration extraction (tacotron2_b200.durations_from_alignments; DESIGN section 6.10): attention maps
// (B, T_mel, T_text) fp32 -> per-symbol frame counts (B, T_text) int64.  Row b reads only
// alignments[b, :mel_lengths[b], :input_lengths[b]] and writes zeros from input_lengths[b] on.
//
//   MAS     the monotonic path from (0, 0) to (L_mel - 1, L_text - 1) that stays on a symbol or advances by one per
//           frame and maximises sum log(max(a, FLT_MIN)), in fp64.  One CTA per row sweeps the frames in order; thread
//           i owns the symbols j = i + m n (n threads, m < K), so a frame's weights are K coalesced loads (issued two
//           frames ahead) and the left neighbour's previous score comes from the lane below by shuffle, or from shared
//           memory at a warp edge (written one frame earlier, double buffered): one barrier per frame.  The backtrack
//           predicate S[t-1][j-1] > S[t-1][j] is one bit per (t, j); each chunk of a warp is one __ballot_sync word, so
//           the map is row-major with ceil(T_text / 32) words per frame, in shared memory when it fits and in the
//           workspace otherwise.  Warp 0 then walks the path back and writes the counts.
//   argmax  one warp per frame takes the first index of the frame's maximum over the row's symbols; one CTA per row
//           then counts the frames per symbol with shared-memory integer atomics (deterministic).
#include <math.h>

#include "common.cuh"

namespace t2 {
namespace {

constexpr int kMasMaxThreads = 256;
constexpr int kArgmaxWarps = 8;                     // frames per CTA of the argmax kernel

// MAS launch shape for T_text symbols (K <= 16 at T_text = 4096): a sweep over the symbols whose bit map has `words`
// words per frame
struct MasPlan : SweepPlan { int words; };
MasPlan mas_plan(int T_mel, int T_text) {
  const int words = (T_text + 31) / 32;
  return {sweep_plan(T_text, kMasMaxThreads, (size_t)T_mel * words * sizeof(uint32_t)), words};
}

struct DurationsWs { uint32_t* bits; int32_t* best; };
void durations_ws_layout(Carve& c, int B, int T_mel, int T_text, int method, DurationsWs* w) {
  w->bits = nullptr;
  w->best = nullptr;
  if (method == T2_DURATIONS_MAS) {
    const MasPlan p = mas_plan(T_mel, T_text);
    if (!p.smem_bits) w->bits = c.take<uint32_t>((size_t)B * T_mel * p.words);     // backtrack bits per row
  } else {
    w->best = c.take<int32_t>((size_t)B * T_mel);                                    // argmax symbol per frame
  }
}

template <int K>
__global__ void __launch_bounds__(kMasMaxThreads) mas_kernel(const float* __restrict__ align,
                                                             const int32_t* __restrict__ in_len,
                                                             const int32_t* __restrict__ mel_len, int T_mel, int T_text,
                                                             int words, uint32_t* __restrict__ gbits,
                                                             int64_t* __restrict__ out) {
  extern __shared__ double smem[];
  const int n = blockDim.x, nw = n >> 5, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.x;
  const int Lt = clamp_length(in_len, b, T_text), Lm = clamp_length(mel_len, b, T_mel);
  int64_t* o = out + (size_t)b * T_text;
  for (int j = tid; j < T_text; j += n)
    if (j >= Lt || Lm < Lt) o[j] = 0;
  if (Lm < Lt) return;                             // no monotonic path through every symbol: zeros
  double* edge = smem;                             // [2][K][nw]: each warp's last lane's score, by frame parity
  uint32_t* bits = gbits ? gbits + (size_t)b * T_mel * words : reinterpret_cast<uint32_t*>(smem + 2 * K * nw);
  const float* a = align + (size_t)b * T_mel * T_text;
  const int D = Lm - Lt;                           // cell (t, j) can still reach the end iff t - D <= j <= t
  const double neg_inf = -INFINITY, flt_min = 1.1754943508222875e-38;    // 2^-126

  double S[K];
  float va[K], vb[K];
#pragma unroll
  for (int m = 0; m < K; ++m) S[m] = neg_inf;
  auto load = [&](float (&v)[K], int t) {
    const int lo = max(0, t - D), hi = min(t, Lt - 1);
    const float* row = a + (size_t)t * T_text;
#pragma unroll
    for (int m = 0; m < K; ++m) {
      const int j = m * n + tid;
      v[m] = (j >= lo && j <= hi) ? __ldg(row + j) : 0.f;
    }
  };
  auto frame = [&](float (&v)[K], int t) {
    const int lo = max(0, t - D), hi = min(t, Lt - 1);
    double c[K];
#pragma unroll
    for (int m = 0; m < K; ++m) c[m] = log(fmax((double)v[m], flt_min));
    if (t + 2 < Lm) load(v, t + 2);
    const double* prev = edge + ((t + 1) & 1) * K * nw;
    double* cur = edge + (t & 1) * K * nw;
#pragma unroll
    for (int m = 0; m < K; ++m) {
      const int j = m * n + tid;
      const double self = S[m], up = __shfl_up_sync(0xffffffffu, self, 1);
      const double left = lane ? up : warp ? prev[m * nw + warp - 1] : m ? prev[(m - 1) * nw + nw - 1] : neg_inf;
      const bool step = left > self;              // the backtrack predicate of (t, j)
      const bool band = j >= lo && j <= hi;
      if (t == 0) {
        S[m] = j == 0 ? c[m] : neg_inf;
      } else {
        S[m] = band ? c[m] + (step ? left : self) : neg_inf;
        const uint32_t word = __ballot_sync(0xffffffffu, step);
        if (lane == 0 && m * n + warp * 32 < Lt) bits[(size_t)t * words + ((m * n) >> 5) + warp] = word;
      }
      if (lane == 31) cur[m * nw + warp] = S[m];
    }
    __syncthreads();
  };
  load(va, 0);
  if (Lm > 1) load(vb, 1);
  for (int t = 0; t < Lm; t += 2) {
    frame(va, t);
    if (t + 1 < Lm) frame(vb, t + 1);
  }

  // warp 0 walks back from (Lm - 1, Lt - 1).  Over 32 frames j falls by at most 31, so lane l first fetches the two
  // words of frame t0 - l that can hold the path's bit, and the walk takes them by shuffle.
  if (warp != 0) return;
  int j = Lt - 1;
  int64_t run = 0;
  for (int t0 = Lm - 1; t0 >= 0; t0 -= 32) {
    const int q = j >> 5, tl = t0 - lane;
    uint32_t whi = 0, wlo = 0;
    if (tl >= 1) {
      whi = bits[(size_t)tl * words + q];
      if (q > 0) wlo = bits[(size_t)tl * words + q - 1];
    }
    const int steps = min(32, t0 + 1);
    for (int s = 0; s < steps; ++s) {
      const int t = t0 - s;
      const uint32_t hi = __shfl_sync(0xffffffffu, whi, s), lo = __shfl_sync(0xffffffffu, wlo, s);
      ++run;
      if (t == 0) break;
      const uint32_t w = (j >> 5) == q ? hi : lo;
      if (j > 0 && (j == t || ((w >> (j & 31)) & 1u))) {
        if (lane == 0) o[j] = run;
        run = 0;
        --j;
      }
    }
  }
  if (lane == 0) o[j] = run;                       // j == 0 here
}

// one warp per frame (b, t < L_mel): the smallest j < L_text holding the frame's maximum over j < L_text
__global__ void argmax_kernel(const float* __restrict__ align, const int32_t* __restrict__ in_len,
                              const int32_t* __restrict__ mel_len, int B, int T_mel, int T_text, int32_t* __restrict__ best) {
  const long f = (long)blockIdx.x * kArgmaxWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= (long)B * T_mel) return;
  const int b = (int)(f / T_mel), t = (int)(f - (long)b * T_mel);
  if (t >= clamp_length(mel_len, b, T_mel)) return;
  const int Lt = clamp_length(in_len, b, T_text);
  const float* row = align + f * T_text;
  float v = -INFINITY;
  int i = Lt;
  for (int j = lane; j < Lt; j += 32) {
    const float x = __ldg(row + j);
    if (x > v || i == Lt) { v = x; i = j; }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, off);
    const int oi = __shfl_xor_sync(0xffffffffu, i, off);
    if (oi < Lt && (i == Lt || ov > v || (ov == v && oi < i))) { v = ov; i = oi; }
  }
  if (lane == 0) best[f] = i;
}

// one CTA per row: durations[b, j] = #frames t < L_mel whose argmax is j (integer counts in shared memory)
__global__ void count_kernel(const int32_t* __restrict__ best, const int32_t* __restrict__ in_len,
                             const int32_t* __restrict__ mel_len, int T_mel, int T_text, int64_t* __restrict__ out) {
  extern __shared__ int cnt[];
  const int b = blockIdx.x;
  const int Lt = clamp_length(in_len, b, T_text), Lm = clamp_length(mel_len, b, T_mel);
  for (int j = threadIdx.x; j < T_text; j += blockDim.x) cnt[j] = 0;
  __syncthreads();
  for (int t = threadIdx.x; t < Lm; t += blockDim.x) {
    const int j = best[(size_t)b * T_mel + t];
    if (j >= 0 && j < Lt) atomicAdd(&cnt[j], 1);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < T_text; j += blockDim.x) out[(size_t)b * T_text + j] = cnt[j];
}

template <int K>
int launch_mas(const T2DurationsArgs* a, const MasPlan& p, uint32_t* gbits, cudaStream_t s) {
  T2_TRY(allow_dynamic_smem(mas_kernel<K>, p.smem_bytes));
  mas_kernel<K><<<a->B, p.threads, p.smem_bytes, s>>>(a->alignments, a->input_lengths, a->mel_lengths, a->T_mel,
                                                       a->T_text, p.words, gbits, a->durations);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

bool durations_sizes_ok(int B, int T_mel, int T_text, int method) {
  return B >= 1 && T_mel >= 1 && T_text >= 1 && T_text <= T2_DURATIONS_MAX_TEXT && (long)B * T_mel <= INT32_MAX &&
         (method == T2_DURATIONS_MAS || method == T2_DURATIONS_ARGMAX);
}

}  // namespace
}  // namespace t2

extern "C" {

size_t t2_durations_workspace_bytes(int32_t B, int32_t T_mel, int32_t T_text, int32_t method) {
  using namespace t2;
  if (!durations_sizes_ok(B, T_mel, T_text, method)) return 0;
  Carve c(nullptr);
  DurationsWs w;
  durations_ws_layout(c, B, T_mel, T_text, method, &w);
  return c.bytes();
}

int t2_durations(const T2DurationsArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->alignments || !a->durations || !a->ws) return fail(T2_ERR_INVALID, "durations: null argument");
  if (!durations_sizes_ok(a->B, a->T_mel, a->T_text, a->method))
    return fail(T2_ERR_INVALID, "durations: bad sizes or method (B %d, T_mel %d, T_text %d in 1..%d, method %d)", a->B,
                a->T_mel, a->T_text, T2_DURATIONS_MAX_TEXT, a->method);
  if (a->ws_bytes < t2_durations_workspace_bytes(a->B, a->T_mel, a->T_text, a->method))
    return fail(T2_ERR_WORKSPACE, "durations workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  Carve c(a->ws);
  DurationsWs w;
  durations_ws_layout(c, a->B, a->T_mel, a->T_text, a->method, &w);
  if (a->method == T2_DURATIONS_ARGMAX) {
    const long frames = (long)a->B * a->T_mel;
    argmax_kernel<<<(unsigned)((frames + kArgmaxWarps - 1) / kArgmaxWarps), 32 * kArgmaxWarps, 0, s>>>(
        a->alignments, a->input_lengths, a->mel_lengths, a->B, a->T_mel, a->T_text, w.best);
    T2_LAUNCH_CHECK();
    count_kernel<<<a->B, 256, a->T_text * sizeof(int), s>>>(w.best, a->input_lengths, a->mel_lengths, a->T_mel, a->T_text,
                                                           a->durations);
    T2_LAUNCH_CHECK();
    return T2_OK;
  }
  const MasPlan p = mas_plan(a->T_mel, a->T_text);
  return with_sweep_k(p.K, [&](auto K) { return launch_mas<decltype(K)::value>(a, p, w.bits, s); });
}

}  // extern "C"
