// Dynamic time warping and mel-cepstra (tacotron2_b200.dtw / mel_cepstral_distortion; DESIGN section 6.12).
//
//   dtw      x (B, D, T_x) and y (B, D, T_y), fp32 or fp64 -> per row the cheapest monotonic path from (0, 0) to
//            (L_x - 1, L_y - 1) with steps (1, 1), (0, 1), (1, 0) over C[i, j] = sqrt(sum_d (x[d, i] - y[d, j])^2),
//            summed in fp64 in the order d = 0 .. D - 1 with no contraction, so every cell equals numpy's sequential sum.
//            D[i, j] = C[i, j] + min(D[i-1, j-1], D[i, j-1], D[i-1, j]); ties go to the diagonal, then (i, j - 1), then
//            (i - 1, j), by the comparisons `left < best`, `up < best` from best = diagonal (NaN never wins).
//            One CTA per row sweeps the anti-diagonals k = i + j in order.  Thread t owns the cells i = t + m n (n
//            threads, m < K) on every diagonal, so along a diagonal consecutive lanes read consecutive frames i of x and
//            consecutive (descending) frames j of y: in the (B, D, T) layout every load of d is coalesced as it stands.
//            The thread keeps its own D on the previous diagonal (the (i, j - 1) predecessor) in a register and its
//            lower neighbour's values on the previous two diagonals ((i - 1, j) and (i - 1, j - 1)) from a shuffle, or
//            from shared memory at a warp edge (written one diagonal earlier, double buffered): one barrier per diagonal.
//            The predecessor is 2 bits per cell, two __ballot_sync words per warp and diagonal, stored per diagonal over
//            the 32-cell blocks of i it touches (`words` pairs per diagonal), in shared memory when the map fits and in
//            the workspace otherwise.  Warp 0 walks the path back 32 diagonals per memory round trip, writes it from the
//            end of the row's path buffer backwards and then moves it to the front, padding with -1.
//   cepstra  per frame, c_k = sum_m table[k][m] mel[m] (table: the orthonormal DCT-II rows k = 1 .. n_cep, built on the
//            host in fp64), summed in fp64 in the order m = 0 .. n_mel - 1; frames past a row's length are 0.
#include <math.h>

#include "common.cuh"

namespace t2 {
namespace {

constexpr int kDtwMaxThreads = 512;
constexpr int kCepThreads = 128;

// launch shape for T_x frames of x (K <= 16 at T_x = 8192): a sweep over the cells i whose predecessor map has `words`
// 32-cell blocks of i per diagonal (a diagonal holds at most min(T_x, T_y) consecutive cells)
struct DtwPlan : SweepPlan { int words; };
DtwPlan dtw_plan(int T_x, int T_y) {
  const int words = std::min((T_x + 31) / 32, (std::min(T_x, T_y) + 31) / 32 + 1);
  return {sweep_plan(T_x, kDtwMaxThreads, (size_t)(T_x + T_y - 1) * words * sizeof(uint2)), words};
}

void dtw_ws_layout(Carve& c, int B, int T_x, int T_y, uint2** bits) {
  const DtwPlan p = dtw_plan(T_x, T_y);
  *bits = p.smem_bits ? nullptr : c.take<uint2>((size_t)B * (T_x + T_y - 1) * p.words);
}

template <typename T, int K, int G = (K < 8 ? K : 8)>
__global__ void __launch_bounds__(kDtwMaxThreads) dtw_kernel(const T* __restrict__ x, const T* __restrict__ y,
                                                             const int32_t* __restrict__ x_len,
                                                             const int32_t* __restrict__ y_len, int D, int T_x,
                                                             int T_y, int words, uint2* __restrict__ gbits,
                                                             double* __restrict__ cost, int64_t* __restrict__ path,
                                                             int64_t* __restrict__ path_len) {
  extern __shared__ double smem[];
  const int n = blockDim.x, nw = n >> 5, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.x;
  const int Lx = clamp_length(x_len, b, T_x), Ly = clamp_length(y_len, b, T_y);
  const T* xb = x + (size_t)b * D * T_x;
  const T* yb = y + (size_t)b * D * T_y;
  double* edge = smem;                              // [2][K][nw]: each warp's last lane's D, by diagonal parity
  uint2* bits = gbits ? gbits + (size_t)b * (T_x + T_y - 1) * words : reinterpret_cast<uint2*>(smem + 2 * K * nw);
  const double inf = INFINITY;

  double S[K], U[K];                                // D[i, k-1-i]; D[i-1, k-2-(i-1)] (the lower neighbour, 2 back)
#pragma unroll
  for (int m = 0; m < K; ++m) S[m] = U[m] = inf;
  for (int k = 0; k < Lx + Ly - 1; ++k) {
    const int lo = max(0, k - Ly + 1), hi = min(k, Lx - 1);
    const double* prev = edge + ((k + 1) & 1) * K * nw;
    double* cur = edge + (k & 1) * K * nw;
    const int q_lo = lo >> 5, q_hi = hi >> 5;
#pragma unroll
    for (int g = 0; g < K; g += G) {                // G cells at a time: their distances, then their D
      double c[G];
      bool valid[G], any = false;
#pragma unroll
      for (int u = 0; u < G; ++u) {
        const int i = (g + u) * n + tid;
        valid[u] = i >= lo && i <= hi;
        any |= valid[u];
        c[u] = 0.0;
      }
      if (__any_sync(0xffffffffu, any)) {
        const T* xd = xb + g * n + tid;             // frame i = (g + u) n + tid of x at d is xd[u n]
        const T* yd = yb + (k - g * n - tid);       // frame j = k - i of y at d is yd[-u n]
#pragma unroll (G >= 8 ? 1 : 4)
        for (int d = 0; d < D; ++d, xd += T_x, yd += T_y) {
#pragma unroll
          for (int u = 0; u < G; ++u)
            if (valid[u]) {
              const double dx = __dsub_rn((double)__ldg(xd + u * n), (double)__ldg(yd - u * n));
              c[u] = __dadd_rn(c[u], __dmul_rn(dx, dx));
            }
        }
      }
#pragma unroll
      for (int u = 0; u < G; ++u) {
        const int m = g + u, i = m * n + tid, j = k - i;
        const double left = S[m], up_lane = __shfl_up_sync(0xffffffffu, left, 1);
        const double up = lane ? up_lane : warp ? prev[m * nw + warp - 1] : m ? prev[(m - 1) * nw + nw - 1] : inf;
        const double diag = U[m];
        U[m] = up;
        int code = 0;
        double v = inf;
        if (valid[u]) {
          const double dist = sqrt(c[u]);
          if (i == 0 && j == 0) {
            v = dist;
          } else if (i == 0) {
            v = __dadd_rn(dist, left);
            code = 1;
          } else if (j == 0) {
            v = __dadd_rn(dist, up);
            code = 2;
          } else {
            double best = diag;
            if (left < best) { best = left; code = 1; }
            if (up < best) { best = up; code = 2; }
            v = __dadd_rn(dist, best);
          }
        }
        S[m] = v;
        const uint32_t w1 = __ballot_sync(0xffffffffu, code == 1), w2 = __ballot_sync(0xffffffffu, code == 2);
        const int q = ((m * n) >> 5) + warp;
        if (lane == 0 && q >= q_lo && q <= q_hi) bits[(size_t)k * words + q - q_lo] = make_uint2(w1, w2);
        if (lane == 31) cur[m * nw + warp] = v;
        if (k == Lx + Ly - 2 && i == Lx - 1) cost[b] = v;
      }
    }
    __syncthreads();
  }

  // warp 0 walks back from (Lx - 1, Ly - 1).  Over 32 diagonals i falls by at most 31, so lane l first fetches the two
  // words of diagonal k0 - l that can hold the path's bits (blocks q and q - 1 of i), and the walk takes them by shuffle.
  if (warp != 0) return;
  const int P = T_x + T_y - 1;
  int64_t* pb = path + (size_t)b * P * 2;
  int i = Lx - 1, j = Ly - 1, N = 0;
  bool done = false;
  while (!done) {
    const int k0 = i + j, q = i >> 5, kl = k0 - lane;
    uint2 whi = make_uint2(0u, 0u), wlo = make_uint2(0u, 0u);
    if (kl >= 1) {
      const int base = max(0, kl - Ly + 1) >> 5;
      if (q - base >= 0 && q - base < words) whi = bits[(size_t)kl * words + q - base];
      if (q - 1 - base >= 0 && q - 1 - base < words) wlo = bits[(size_t)kl * words + q - 1 - base];
    }
    for (;;) {
      const int l = k0 - (i + j);
      if (l >= 32) break;
      if (lane == 0) {
        pb[2 * (P - 1 - N)] = i;
        pb[2 * (P - 1 - N) + 1] = j;
      }
      ++N;
      if (i == 0 && j == 0) { done = true; break; }
      const uint32_t h1 = __shfl_sync(0xffffffffu, whi.x, l), h2 = __shfl_sync(0xffffffffu, whi.y, l);
      const uint32_t l1 = __shfl_sync(0xffffffffu, wlo.x, l), l2 = __shfl_sync(0xffffffffu, wlo.y, l);
      const bool own = (i >> 5) == q;
      const uint32_t b1 = ((own ? h1 : l1) >> (i & 31)) & 1u, b2 = ((own ? h2 : l2) >> (i & 31)) & 1u;
      const int code = i == 0 ? 1 : j == 0 ? 2 : b1 ? 1 : b2 ? 2 : 0;
      if (code != 1) --i;
      if (code != 2) --j;
    }
  }
  __syncwarp();
  // move the N cells from [P - N, P) to [0, N) in ascending chunks (a chunk's sources lie at or above its targets and
  // above every earlier chunk's targets), and pad [N, P) with -1
  for (int t0 = 0; t0 < P; t0 += 32) {
    const int t = t0 + lane;
    int64_t a = -1, c = -1;
    if (t < N) {
      a = pb[2 * (P - N + t)];
      c = pb[2 * (P - N + t) + 1];
    }
    __syncwarp();
    if (t < P) {
      pb[2 * t] = a;
      pb[2 * t + 1] = c;
    }
    __syncwarp();
  }
  if (lane == 0) path_len[b] = N;
}

template <typename T>
__global__ void __launch_bounds__(kCepThreads) cepstra_kernel(const T* __restrict__ mel, const int32_t* __restrict__ len,
                                                              int n_mel, int T_f, const double* __restrict__ table,
                                                              int n_cep, double* __restrict__ cep) {
  const int b = blockIdx.y, t = blockIdx.x * kCepThreads + threadIdx.x;
  if (t >= T_f) return;
  const int L = clamp_length(len, b, T_f);
  const T* col = mel + (size_t)b * n_mel * T_f + t;
  double* out = cep + (size_t)b * n_cep * T_f + t;
  for (int k = 0; k < n_cep; ++k) {
    double s = 0.0;
    if (t < L) {
      const double* row = table + (size_t)k * n_mel;
      for (int m = 0; m < n_mel; ++m) s = __dadd_rn(s, __dmul_rn(__ldg(row + m), (double)__ldg(col + (size_t)m * T_f)));
    }
    out[(size_t)k * T_f] = s;
  }
}

template <typename T, int K>
int launch_dtw(const T2DtwArgs* a, const DtwPlan& p, uint2* gbits, cudaStream_t s) {
  T2_TRY(allow_dynamic_smem(dtw_kernel<T, K>, p.smem_bytes));
  dtw_kernel<T, K><<<a->B, p.threads, p.smem_bytes, s>>>(
      static_cast<const T*>(a->x), static_cast<const T*>(a->y), a->x_lengths, a->y_lengths, a->D, a->T_x, a->T_y,
      p.words, gbits, a->cost, a->path, a->path_lengths);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int dtw_sizes_status(int B, int D, int T_x, int T_y, int dtype) {
  if (B < 1 || D < 1 || T_x < 1 || T_y < 1 || (dtype != T2_DTW_F32 && dtype != T2_DTW_F64)) return T2_ERR_INVALID;
  if (D > T2_DTW_MAX_DIM || T_x > T2_DTW_MAX_FRAMES || T_y > T2_DTW_MAX_FRAMES) return T2_ERR_UNSUPPORTED;
  return T2_OK;
}

}  // namespace
}  // namespace t2

extern "C" {

size_t t2_dtw_workspace_bytes(int32_t B, int32_t D, int32_t T_x, int32_t T_y, int32_t dtype) {
  using namespace t2;
  if (dtw_sizes_status(B, D, T_x, T_y, dtype) != T2_OK) return 0;
  Carve c(nullptr);
  uint2* bits;
  dtw_ws_layout(c, B, T_x, T_y, &bits);
  return c.bytes();
}

int t2_dtw(const T2DtwArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->x || !a->y || !a->cost || !a->path || !a->path_lengths || !a->ws)
    return fail(T2_ERR_INVALID, "dtw: null argument");
  const int st = dtw_sizes_status(a->B, a->D, a->T_x, a->T_y, a->dtype);
  if (st != T2_OK)
    return fail(st, "dtw: bad sizes or dtype (B %d, D %d in 1..%d, T_x %d and T_y %d in 1..%d, dtype %d)", a->B, a->D,
                T2_DTW_MAX_DIM, a->T_x, a->T_y, T2_DTW_MAX_FRAMES, a->dtype);
  if (a->ws_bytes < t2_dtw_workspace_bytes(a->B, a->D, a->T_x, a->T_y, a->dtype))
    return fail(T2_ERR_WORKSPACE, "dtw workspace too small");
  Carve c(a->ws);
  uint2* bits;
  dtw_ws_layout(c, a->B, a->T_x, a->T_y, &bits);
  const DtwPlan p = dtw_plan(a->T_x, a->T_y);
  cudaStream_t s = (cudaStream_t)stream;
  return with_sweep_k(p.K, [&](auto K) {
    return a->dtype == T2_DTW_F32 ? launch_dtw<float, decltype(K)::value>(a, p, bits, s)
                                  : launch_dtw<double, decltype(K)::value>(a, p, bits, s);
  });
}

int t2_mel_cepstra(const void* mel, int32_t dtype, const int32_t* lengths, int32_t B, int32_t n_mel, int32_t T,
                   const double* table, int32_t n_cep, double* cep, void* stream) {
  using namespace t2;
  if (!mel || !table || !cep) return fail(T2_ERR_INVALID, "mel_cepstra: null argument");
  const int st = dtw_sizes_status(B, n_mel, T, 1, dtype);
  if (st != T2_OK || n_cep < 1 || n_cep >= n_mel || B > 65535)
    return fail(st != T2_OK ? st : T2_ERR_INVALID,
                "mel_cepstra: bad sizes or dtype (B %d in 1..65535, n_mel %d in 2..%d, T %d in 1..%d, n_cep %d in "
                "1..n_mel - 1, dtype %d)", B, n_mel, T2_DTW_MAX_DIM, T, T2_DTW_MAX_FRAMES, n_cep, dtype);
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((T + kCepThreads - 1) / kCepThreads, B);
  if (dtype == T2_DTW_F32)
    cepstra_kernel<float><<<grid, kCepThreads, 0, s>>>(static_cast<const float*>(mel), lengths, n_mel, T, table, n_cep,
                                                       cep);
  else
    cepstra_kernel<double><<<grid, kCepThreads, 0, s>>>(static_cast<const double*>(mel), lengths, n_mel, T, table,
                                                        n_cep, cep);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
