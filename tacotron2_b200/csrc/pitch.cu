// Pitch targets (tacotron2_b200.pyin / average_by_durations; DESIGN section 6.11).
//
//   pyin   librosa 0.10's pYIN (center=True, pad_mode="constant") over a ragged batch of clips, in fp64.  Two kernels:
//          pyin_frame_kernel, one CTA per (frame, clip): stages the frame's samples (its own zeros past the clip) in
//          shared memory, takes the difference function (the ACF as direct sums, e[tau] as a difference of the serial
//          cumulative sum of squares -- numpy's cumsum order), the cumulative mean normalised difference, then warp 0
//          finds the troughs, their threshold probabilities, parabolic shifts and pitch bins, and writes the frame's
//          voiced observations (sparse, log(p + tiny), ascending bin), its unvoiced log observation and voiced_prob.
//          pyin_viterbi_kernel, one CTA per clip, sequential over frames: librosa.sequence.viterbi over 2 n_bins states
//          with the band of the local-triangle transition matrix read from a host table, predecessors as int16 in the
//          workspace, then a walk back from the last frame.
//   average_by_durations   one CTA per row: the mean of each symbol's non-zero, non-NaN frame values, summed in fp64 in
//          frame order.
#include <math.h>

#include "common.cuh"

namespace t2 {
namespace {

constexpr int kFrameThreads = 256;
constexpr int kViterbiThreads = 1024;
constexpr int kAverageThreads = 256;
constexpr double kTiny = 2.2250738585072014e-308;      // numpy's finfo(float64).tiny

__host__ __device__ inline int pyin_frames(int n, int hop) { return 1 + n / hop; }
__host__ __device__ inline int pyin_lags(const T2PyinArgs& a) { return a.max_period - a.min_period + 1; }
// troughs cannot be neighbours (strict left / non-strict right minima), so a frame has at most ceil(lags / 2)
__host__ __device__ inline int pyin_max_troughs(const T2PyinArgs& a) { return (pyin_lags(a) + 1) / 2; }

struct PyinWs { double *log_u, *logp; int32_t* count; int16_t *bins, *ptr; };
void pyin_ws_layout(Carve& c, const T2PyinArgs& a, PyinWs* w) {
  const size_t BF = (size_t)a.B * pyin_frames(a.n, a.hop_length), K = pyin_max_troughs(a);
  w->log_u = c.take<double>(BF);                        // per frame: log((1 - voiced_prob) / n_bins + tiny)
  w->logp = c.take<double>(BF * K);                     // per frame: the voiced observations' log(p + tiny) ...
  w->count = c.take<int32_t>(BF);                       // ... how many there are ...
  w->bins = c.take<int16_t>(BF * K);                    // ... and their bins, ascending
  w->ptr = c.take<int16_t>(BF * 2 * a.n_bins);          // Viterbi predecessors
}

size_t frame_smem_bytes(const T2PyinArgs& a) {
  const int fl = a.frame_length, lags = pyin_lags(a);
  return sizeof(double) * (2 * (size_t)fl + (a.max_period + 1) + lags + (a.n_bins + 1)) +
         sizeof(int) * ((size_t)pyin_max_troughs(a) * 2 + (a.n_bins + 1) + 2 * (a.n_thresholds + 1));
}

size_t viterbi_smem_bytes(const T2PyinArgs& a) {
  const size_t n = a.n_bins;
  return sizeof(double) * (4 * n + n + 8 * n) + sizeof(int) * 8 * n + 64;
}

__global__ void __launch_bounds__(kFrameThreads) pyin_frame_kernel(T2PyinArgs a, PyinWs w) {
  extern __shared__ double sm[];
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  const int fl = a.frame_length, W = a.win_length, maxp = a.max_period, minp = a.min_period, lags = pyin_lags(a);
  const int nb = a.n_bins, nthr = a.n_thresholds, K = pyin_max_troughs(a);
  const int F = pyin_frames(a.n, a.hop_length), L = clamp_length(a.lengths, b, a.n);
  const size_t bf = (size_t)b * F + f;
  if (f >= pyin_frames(L, a.hop_length)) {             // past the row's end: no observations, voiced_prob 0
    if (tid == 0) { w.count[bf] = 0; w.log_u[bf] = 0.0; a.voiced_prob[bf] = 0.0; }
    return;
  }
  double* x = sm;                                        // [fl] the frame
  double* cs = x + fl;                                   // [fl] cumulative sum of squares
  double* d = cs + fl;                                   // [maxp + 1] difference function, then its cumulative sum
  double* yin = d + maxp + 1;                            // [lags]
  double* obs = yin + lags;                              // [nb + 1] the frame's voiced observations by bin
  int* tr = reinterpret_cast<int*>(obs + nb + 1);        // [K] trough lags
  int* tk = tr + K;                                      // [K] first threshold each trough lies below
  int* win = tk + K;                                     // [nb + 1] the largest trough holding each bin
  int* hist = win + nb + 1;                              // [nthr + 1] troughs per first threshold, then n_troughs
  int* before = hist + nthr + 1;                         // [nthr + 1] troughs of earlier chunks below each threshold

  const float* yb = a.y + (size_t)b * a.n;
  const long g0 = (long)f * a.hop_length - fl / 2;
  for (int m = tid; m < fl; m += blockDim.x) {
    const long g = g0 + m;
    x[m] = (g >= 0 && g < L) ? (double)yb[g] : 0.0;
  }
  for (int k = tid; k <= nb; k += blockDim.x) { obs[k] = 0.0; win[k] = -1; }
  for (int k = tid; k <= nthr; k += blockDim.x) { hist[k] = 0; before[k] = 0; }
  __syncthreads();
  // acf[tau] = sum_{j=1..W} x[j] x[j + tau] by the other threads; numpy's serial cumsum of x^2 by the last one
  const int last = blockDim.x - 1;
  if (tid == last) {
    double acc = 0.0;
    for (int m = 0; m < fl; ++m) { acc = __dadd_rn(acc, __dmul_rn(x[m], x[m])); cs[m] = acc; }
  } else {
    for (int tau = tid; tau <= maxp; tau += last) {
      double s = 0.0;
      const double* xt = x + tau;
      for (int j = 1; j <= W; ++j) s = fma(x[j], xt[j], s);
      d[tau] = s;
    }
  }
  __syncthreads();
  const double e0 = [&] { const double e = __dsub_rn(cs[W], cs[0]); return fabs(e) < 1e-6 ? 0.0 : e; }();
  for (int tau = tid; tau <= maxp; tau += blockDim.x) {
    double acf = d[tau], e = __dsub_rn(cs[tau + W], cs[tau]);
    if (fabs(acf) < 1e-6) acf = 0.0;
    if (fabs(e) < 1e-6) e = 0.0;
    d[tau] = __dsub_rn(__dadd_rn(e0, e), 2.0 * acf);
  }
  __syncthreads();
  // yin[tau - minp] = d[tau] / (mean(d[1..tau]) + tiny), the running sum in numpy's order
  if (tid == 0) {
    double acc = 0.0;
    for (int tau = 1; tau <= maxp; ++tau) {
      const double dt = d[tau];
      acc = __dadd_rn(acc, dt);
      if (tau >= minp) yin[tau - minp] = __ddiv_rn(dt, __dadd_rn(__ddiv_rn(acc, (double)tau), kTiny));
    }
  }
  __syncthreads();
  if (tid >= 32) return;

  // ---- warp 0: troughs, their probabilities and the frame's observations (librosa's __pyin_helper) ----
  const unsigned lt = (1u << lane) - 1u;
  int nt = 0;
  for (int c = 0; c < lags; c += 32) {
    const int i = c + lane;
    bool t = false;
    if (i < lags) {
      const double yi = yin[i];
      if (i == 0) t = yi < yin[1];
      else if (i == lags - 1) t = yi < yin[i - 1];
      else t = yi < yin[i - 1] && yi <= yin[i + 1];
    }
    const unsigned m = __ballot_sync(0xffffffffu, t);
    if (t) {
      const int p = nt + __popc(m & lt);
      tr[p] = i;
      // thresholds at or below the height: the count of thresholds it does not lie below
      const double h = yin[i];
      int lo = 0, hi = nthr;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (h < a.thresholds[mid]) hi = mid; else lo = mid + 1; }
      tk[p] = lo;
      atomicAdd(&hist[lo], 1);
    }
    nt += __popc(m);
  }
  __syncwarp();
  if (lane == 0) {                                       // n_troughs[k] = #troughs below threshold k
    int acc = 0;
    for (int k = 0; k < nthr; ++k) { acc += hist[k]; hist[k] = acc; }
  }
  __syncwarp();
  // the global minimum trough: the first with the smallest height
  double hmin = INFINITY;
  int gmin = nt;
  for (int p = lane; p < nt; p += 32) {
    const double h = yin[tr[p]];
    if (h < hmin || gmin == nt) { hmin = h; gmin = p; }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double oh = __shfl_xor_sync(0xffffffffu, hmin, off);
    const int og = __shfl_xor_sync(0xffffffffu, gmin, off);
    if (og < nt && (gmin == nt || oh < hmin || (oh == hmin && og < gmin))) { hmin = oh; gmin = og; }
  }
  const double log_tiny = a.log_tiny;
  for (int c = 0; c < nt; c += 32) {
    const int p = c + lane;
    const bool valid = p < nt;
    const int kp = valid ? tk[p] : nthr;
    double prob = 0.0;
    for (int k = 0; k < nthr; ++k) {
      const bool below = valid && k >= kp;
      const unsigned m = __ballot_sync(0xffffffffu, below);
      if (m == 0) continue;
      const int b0 = before[k];
      if (below) {
        const int N = hist[k], pos = b0 + __popc(m & lt);
        prob = __dadd_rn(prob, __dmul_rn(a.boltzmann[(size_t)N * (N - 1) / 2 + pos], a.beta_probs[k]));
      }
      __syncwarp();
      if (lane == 0) before[k] = b0 + __popc(m);
      __syncwarp();
    }
    if (p == gmin) prob = __dadd_rn(prob, __dmul_rn(a.no_trough_prob, a.beta_prefix[kp]));
    int bin = -1;
    if (valid && prob != 0.0) {                          // a candidate: the pitch bin of its refined period
      const int i = tr[p];
      double shift = 0.0;
      if (i > 0 && i < lags - 1) {
        const double ya = __dsub_rn(__dadd_rn(yin[i + 1], yin[i - 1]), 2.0 * yin[i]);
        const double yb2 = __ddiv_rn(__dsub_rn(yin[i + 1], yin[i - 1]), 2.0);
        if (!(fabs(yb2) >= fabs(ya))) shift = __ddiv_rn(-yb2, ya);
      }
      const double period = __dadd_rn((double)(minp + i), shift);
      const double f0 = __ddiv_rn(__ddiv_rn((double)a.sr, period), a.fmin);
      const double idx = __dmul_rn((double)(12 * a.bins_per_semitone), log2(f0));
      bin = (int)fmin(fmax(rint(idx), 0.0), (double)nb);
      atomicMax(&win[bin], p);                           // the largest lag wins a shared bin
    }
    __syncwarp();
    if (bin >= 0 && bin < nb && win[bin] == p) obs[bin] = prob;
  }
  __syncwarp();
  // voiced_prob = clip(sum of the voiced observations in bin order); the observations out in the same order
  double vp = 0.0;
  int cnt = 0;
  double* logp = w.logp + bf * K;
  int16_t* bins = w.bins + bf * K;
  for (int c = 0; c < nb; c += 32) {
    const int k = c + lane;
    const double o = k < nb ? obs[k] : 0.0;
    unsigned m = __ballot_sync(0xffffffffu, o != 0.0);
    if (o != 0.0) {
      const int q = cnt + __popc(m & lt);
      logp[q] = log(o + kTiny);
      bins[q] = (int16_t)k;
    }
    while (m) {
      const int src = __ffs(m) - 1;
      vp = __dadd_rn(vp, __shfl_sync(0xffffffffu, o, src));
      m &= m - 1;
    }
    cnt += __popc(__ballot_sync(0xffffffffu, o != 0.0));
  }
  if (lane == 0) {
    vp = fmin(fmax(vp, 0.0), 1.0);
    const double u = __ddiv_rn(1.0 - vp, (double)nb);
    w.log_u[bf] = u == 0.0 ? log_tiny : log(u + kTiny);
    w.count[bf] = cnt;
    a.voiced_prob[bf] = vp;
  }
}

// first index of the larger value: (v, i) replaces (bv, bi) when v > bv or (v == bv and i < bi)
__device__ __forceinline__ void take_best(double v, int i, double& bv, int& bi) {
  if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
}

// librosa.sequence.viterbi over 2 nb states, one CTA per clip.  Out of the band |bin(i) - bin(j)| <= h the transition is
// log(0 + tiny) = log_tiny for every (i, j), so the out-of-band candidates of destination j are s[i] = v[i] + log_tiny
// over four index ranges: [0, lo), (hi, nb), [nb, nb + lo), (nb + hi, 2 nb) with lo = bin(j) - h, hi = bin(j) + h.  Their
// first-index maxima come from per-frame prefix / suffix scans of s in each half; the in-band predecessors are computed
// one by one from the table; visiting the pieces in index order with a strict > keeps numpy argmax's first index.
__global__ void __launch_bounds__(kViterbiThreads) pyin_viterbi_kernel(T2PyinArgs a, PyinWs w) {
  extern __shared__ double sm[];
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int nb = a.n_bins, S = 2 * nb, h = a.width / 2, bw = 2 * h + 1, K = pyin_max_troughs(a);
  const int F = pyin_frames(a.n, a.hop_length), Fb = pyin_frames(clamp_length(a.lengths, b, a.n), a.hop_length);
  double* v = sm;                                        // [2][S] scores of the previous / current frame
  double* lobs = v + 2 * S;                              // [nb] the frame's voiced log observations
  double* sv = lobs + nb;                                // [2][4 nb] scan values: prefix / suffix of each half
  int* si = reinterpret_cast<int*>(sv + 8 * nb);         // [2][4 nb] their indices
  __shared__ double red_v[32];
  __shared__ int red_i[32];
  const size_t f0i = (size_t)b * F;
  const double log_tiny = a.log_tiny;
  const double* T = a.log_trans;                         // [2][bw][nb]: 0 within a voicing half, 1 across

  for (int k = tid; k < nb; k += nt) lobs[k] = log_tiny;
  __syncthreads();
  {
    const int c = w.count[f0i];
    for (int q = tid; q < c; q += nt) lobs[w.bins[f0i * K + q]] = w.logp[f0i * K + q];
  }
  __syncthreads();
  for (int j = tid; j < S; j += nt)
    v[j] = __dadd_rn(j < nb ? lobs[j] : w.log_u[f0i], j < nb ? log_tiny : a.log_init_unvoiced);
  __syncthreads();
  int cur = 0;
  for (int t = 1; t < Fb; ++t) {
    const size_t ft = f0i + t;
    const double* vp = v + cur * S;
    double* vn = v + (cur ^ 1) * S;
    // scan inputs; the previous frame's observations back to log_tiny
    for (int e = tid; e < 4 * nb; e += nt) {
      const int arr = e / nb, k = e - arr * nb, i = (arr >> 1) * nb + k;
      sv[e] = __dadd_rn(vp[i], log_tiny);
      si[e] = i;
    }
    {
      const size_t fp = ft - 1;
      const int c = w.count[fp];
      for (int q = tid; q < c; q += nt) lobs[w.bins[fp * K + q]] = log_tiny;
    }
    __syncthreads();
    {
      const int c = w.count[ft];
      for (int q = tid; q < c; q += nt) lobs[w.bins[ft * K + q]] = w.logp[ft * K + q];
    }
    // Hillis-Steele: arrays 0 / 2 prefix maxima, 1 / 3 suffix maxima, first index on ties
    int src = 0;
    for (int dlt = 1; dlt < nb; dlt <<= 1) {
      const double* ov = sv + src * 4 * nb;
      const int* oi = si + src * 4 * nb;
      double* nv = sv + (src ^ 1) * 4 * nb;
      int* ni = si + (src ^ 1) * 4 * nb;
      for (int e = tid; e < 4 * nb; e += nt) {
        const int arr = e / nb, k = e - arr * nb;
        double bv = ov[e];
        int bi = oi[e];
        const int o = (arr & 1) ? k + dlt : k - dlt;
        if (o >= 0 && o < nb) take_best(ov[e - k + o], oi[e - k + o], bv, bi);
        nv[e] = bv;
        ni[e] = bi;
      }
      src ^= 1;
      __syncthreads();
    }
    if (nb == 1) __syncthreads();
    const double* pv = sv + src * 4 * nb;
    const int* pi = si + src * 4 * nb;
    const double lu = w.log_u[ft];
    int16_t* ptr = w.ptr + ft * S;
    for (int j = tid; j < S; j += nt) {
      const int hj = j >= nb, jb = j - hj * nb, lo = jb - h, hi = jb + h;
      double bv = -INFINITY;
      int bi = S;
#pragma unroll
      for (int hs = 0; hs < 2; ++hs) {
        const double* Tb = T + (size_t)(hs != hj) * bw * nb + jb;
        if (lo > 0) take_best(pv[(2 * hs) * nb + lo - 1], pi[(2 * hs) * nb + lo - 1], bv, bi);
        const int k0 = max(0, -lo), k1 = min(bw, nb - lo);
        const double* vs = vp + hs * nb + lo;
        for (int k = k0; k < k1; ++k) {
          const double s = __dadd_rn(vs[k], Tb[(size_t)k * nb]);
          if (s > bv) { bv = s; bi = hs * nb + lo + k; }
        }
        if (hi < nb - 1) take_best(pv[(2 * hs + 1) * nb + hi + 1], pi[(2 * hs + 1) * nb + hi + 1], bv, bi);
      }
      vn[j] = __dadd_rn(hj ? lu : lobs[jb], bv);
      ptr[j] = (int16_t)bi;
    }
    cur ^= 1;
    __syncthreads();
  }
  // the last frame's first argmax, then the walk back by thread 0
  const double* vl = v + cur * S;
  double bv = -INFINITY;
  int bi = S;
  for (int j = tid; j < S; j += nt) take_best(vl[j], j, bv, bi);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    take_best(ov, oi, bv, bi);
  }
  if ((tid & 31) == 0) { red_v[tid >> 5] = bv; red_i[tid >> 5] = bi; }
  __syncthreads();
  for (int f = Fb + tid; f < F; f += nt) { a.f0[f0i + f] = 0.0; a.voiced_flag[f0i + f] = 0; }
  if (tid != 0) return;
  for (int q = 1; q < (nt + 31) / 32; ++q) take_best(red_v[q], red_i[q], red_v[0], red_i[0]);
  int s = red_i[0];
  for (int t = Fb - 1; t >= 0; --t) {
    const bool voiced = s < nb;
    a.f0[f0i + t] = voiced ? a.freqs[s] : a.fill_na;
    a.voiced_flag[f0i + t] = voiced;
    if (t > 0) s = w.ptr[(f0i + t) * S + s];
  }
}

// one CTA per row: out[b, j] = mean of values[b, f] over f in [cum_j, cum_{j+1}) with values neither 0 nor NaN
__global__ void __launch_bounds__(kAverageThreads) average_kernel(const double* __restrict__ values,
                                                                  const int64_t* __restrict__ dur, int F, int T,
                                                                  float* __restrict__ out) {
  __shared__ long long carry_s[kAverageThreads / 32];
  __shared__ long long carry;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* vb = values + (size_t)b * F;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int c = 0; c < T; c += blockDim.x) {
    const int j = c + tid;
    const long long d = j < T ? max((long long)dur[(size_t)b * T + j], 0LL) : 0LL;
    long long incl = d;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const long long o = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += o;
    }
    if (lane == 31) carry_s[warp] = incl;
    __syncthreads();
    long long base = carry;
    for (int q = 0; q < warp; ++q) base += carry_s[q];
    const long long end = base + incl, start = end - d;
    if (j < T) {
      double s = 0.0;
      int n = 0;
      for (long long f = start; f < min(end, (long long)F); ++f) {
        const double x = vb[f];
        if (x != 0.0 && !isnan(x)) { s += x; ++n; }
      }
      out[(size_t)b * T + j] = n ? (float)(s / n) : 0.f;
    }
    __syncthreads();
    if (tid == blockDim.x - 1) carry = end;
    __syncthreads();
  }
}

bool pyin_sizes_ok(const T2PyinArgs& a) {
  const long F = a.n >= 1 && a.hop_length >= 1 ? pyin_frames(a.n, a.hop_length) : 0;
  return a.B >= 1 && a.n >= 1 && a.sr >= 1 && a.frame_length >= 2 && a.frame_length <= T2_PYIN_MAX_FRAME &&
         a.win_length >= 1 && a.win_length < a.frame_length && a.hop_length >= 1 && a.min_period >= 1 &&
         a.max_period > a.min_period && a.max_period <= a.frame_length - a.win_length - 1 && a.n_thresholds >= 1 &&
         a.n_thresholds <= T2_PYIN_MAX_THRESHOLDS && a.n_bins >= 1 && a.n_bins <= T2_PYIN_MAX_BINS && a.width >= 1 &&
         a.bins_per_semitone >= 1 && (long)a.B * F <= INT32_MAX && a.fmin > 0;
}

}  // namespace
}  // namespace t2

extern "C" {

size_t t2_pyin_workspace_bytes(const T2PyinArgs* a) {
  using namespace t2;
  if (!a || !pyin_sizes_ok(*a)) return 0;
  Carve c(nullptr);
  PyinWs w;
  pyin_ws_layout(c, *a, &w);
  return c.bytes();
}

int t2_pyin(const T2PyinArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->y || !a->f0 || !a->voiced_flag || !a->voiced_prob || !a->ws || !a->thresholds || !a->beta_probs ||
      !a->beta_prefix || !a->boltzmann || !a->log_trans || !a->freqs)
    return fail(T2_ERR_INVALID, "pyin: null argument");
  if (!pyin_sizes_ok(*a))
    return fail(T2_ERR_INVALID,
                "pyin: bad sizes (B %d, n %d, sr %d, frame_length %d in 2..%d, win_length %d, hop_length %d, periods "
                "%d..%d, n_thresholds %d in 1..%d, n_bins %d in 1..%d, width %d, bins_per_semitone %d)",
                a->B, a->n, a->sr, a->frame_length, T2_PYIN_MAX_FRAME, a->win_length, a->hop_length, a->min_period,
                a->max_period, a->n_thresholds, T2_PYIN_MAX_THRESHOLDS, a->n_bins, T2_PYIN_MAX_BINS, a->width,
                a->bins_per_semitone);
  if (a->ws_bytes < t2_pyin_workspace_bytes(a)) return fail(T2_ERR_WORKSPACE, "pyin workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  Carve c(a->ws);
  PyinWs w;
  pyin_ws_layout(c, *a, &w);
  const size_t fsm = frame_smem_bytes(*a), vsm = viterbi_smem_bytes(*a);
  T2_TRY(allow_dynamic_smem(pyin_frame_kernel, fsm));
  T2_TRY(allow_dynamic_smem(pyin_viterbi_kernel, vsm));
  const int F = pyin_frames(a->n, a->hop_length);
  pyin_frame_kernel<<<dim3(F, a->B), kFrameThreads, fsm, s>>>(*a, w);
  T2_LAUNCH_CHECK();
  pyin_viterbi_kernel<<<a->B, kViterbiThreads, vsm, s>>>(*a, w);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

int t2_average_by_durations(const double* values, const int64_t* durations, int32_t B, int32_t F, int32_t T_text,
                            float* out, void* stream) {
  using namespace t2;
  if (!values || !durations || !out) return fail(T2_ERR_INVALID, "average_by_durations: null argument");
  if (B < 1 || F < 1 || T_text < 1)
    return fail(T2_ERR_INVALID, "average_by_durations: bad sizes (B %d, F %d, T_text %d)", B, F, T_text);
  average_kernel<<<B, kAverageThreads, 0, (cudaStream_t)stream>>>(values, durations, F, T_text, out);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
