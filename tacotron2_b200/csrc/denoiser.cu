// WaveGlow denoiser (waveglow/denoiser.py: Denoiser.forward over stft.py:69-136 and audio_processing.py:7-56) on sm_90a.
//
// Both transforms are convolutions with kernel 1024 and stride 256, i.e. 4 taps of one 256-sample block each, so each
// is one implicit GEMM of wg_gemm.cuh whose rows are 256-sample blocks:
//
//   pack (CUDA cores)   reflect-pad every row at its own end and write the padded signal as k8 planes, one plane row
//                       per 256-sample block (32 groups of 8 samples).
//   forward             rows = frames; K = padded blocks f ... f + 3 (4 segments, row shifts -1 ... 2) x 256 samples;
//                       N = the 1026 basis rows reordered so that each 256-column tile holds the real and imaginary rows
//                       of the same 128 bins (5 tiles).  The epilogue (EPI_SPECTRAL) takes the magnitude, subtracts
//                       strength * bias, clamps at 0, rescales (re, im) and writes them as the next GEMM's planes.
//   inverse             rows = output blocks; K = the 4 frames that overlap a block (segments at row shifts 0 ... 3,
//                       each against its 256 columns of the inverse basis) x 1088 spectrum channels; N = 256.  The
//                       overlap-add happens in the accumulator; the epilogue (EPI_OVERLAP) divides by window_sumsquare,
//                       multiplies by 4, trims and writes fp32 audio.
//
// Rows of one sequence b: q = b * span + t, span = F + 4 for F = n / 256 + 1 frames.  The padded block i sits at plane
// row 1 + b * span + i; spectrum row t holds frame t - 1 (t = 0 and t > F are zero frames); output row t is block t.
// Only the fp32-grade tier (split fp16, 3 MMAs) exists: the reference denoises in fp32.
//
// The public STFT (stft.py:69-141) and Griffin-Lim (audio_processing.py:59-75) run on the same two GEMMs and planes:
//   transform     row scale, pack, forward with EPI_MAGPHASE (fp32 magnitude and atan2 phase)
//   inverse       spec_pack_kernel ((magnitude, phase) -> spectrum planes), inverse
//   Griffin-Lim   spec_pack_kernel, inverse, then per iteration: pack (of the previous signal), forward with
//                 EPI_PROJECT (the target magnitude on the current phase), inverse: 3 n_iters + 2 launches.
// Their operands are scaled per row by a power of two taken on the device from the row's largest target magnitude (or
// sample): the stored spectrum then peaks in [1, 2) and audio in [0.5, 1), the ranges in which the denoiser runs
// unit-scale audio, whatever the caller's scale.  The fp32 outputs undo it exactly.
#include <cooperative_groups.h>
#include <math.h>
#include <string.h>
#include <algorithm>

#include "conv_tc.h"
#include "denoiser.h"
#include "wg_gemm.cuh"

struct T2Denoiser {
  float* fwd = nullptr;          // forward basis (1026, 1024) fp32: the one-frame bias kernel reads it
  uint8_t* fwd_img = nullptr;    // forward GEMM weights, (1280, 1024) in tile order
  uint8_t* inv_img = nullptr;    // inverse GEMM weights, (256, 4 x 1088)
  double* wsq = nullptr;         // squared periodic Hann window (1024), as window_sumsquare builds it
  float* tmp = nullptr;          // fp32 staging of the matrix being packed
};

namespace t2 {
namespace {

constexpr int kFilter = 1024, kHop = 256, kBasisRows = 2 * kBins;
constexpr int kFwdTiles = 5, kFwdN = kFwdTiles * 256;          // 5 x 128 bin slots >= 513 bins
constexpr int kSpecCh = kSpecGroups * 8;                        // 1088 = 17 chunks
constexpr int kInvK = 4 * kSpecCh;
constexpr int kBlkGroups = kHop / 8;
// Reach: output block k depends on the frames k - 1 ... k + 2, and frame f on the input blocks f - 2 ... f + 1, so on
// the input blocks k - 3 ... k + 3.
constexpr int kHalo = 3;
constexpr int kPassesFp32 = 3;

// forward weights: packed row nn = tile * 256 + h * 128 + c is basis row bin (h = 0, real) or 513 + bin (h = 1,
// imaginary) of bin = tile * 128 + c; rows of bins >= 513 are zero
__global__ void build_fwd_kernel(const float* __restrict__ fwd, float* __restrict__ w) {
  const int nn = blockIdx.x, tile = nn >> 8, h = (nn >> 7) & 1, bin = tile * 128 + (nn & 127);
  const int src = bin < kBins ? h * kBins + bin : -1;
  for (int k = threadIdx.x; k < kFilter; k += blockDim.x)
    w[(long)nn * kFilter + k] = src >= 0 ? fwd[(long)src * kFilter + k] : 0.f;
}

// inverse weights: row p (output sample of a block), k = sh * 1088 + ch.  Segment sh reads frame t - 1 + sh for output
// block t, which lands 256 (3 - sh) samples into that frame.  Channel ch < 520 is the real part of bin ch, channel
// 520 + bin the imaginary part (the spectrum plane layout of EPI_SPECTRAL); the padding channels are zero.  Packed
// times kInvBasisScale.
__global__ void build_inv_kernel(const float* __restrict__ inv, float* __restrict__ w) {
  const int p = blockIdx.x;
  for (int k = threadIdx.x; k < kInvK; k += blockDim.x) {
    const int sh = k / kSpecCh, ch = k % kSpecCh;
    int src = -1;
    if (ch < 8 * kImGroup0) src = ch < kBins ? ch : -1;
    else if (ch - 8 * kImGroup0 < kBins) src = kBins + ch - 8 * kImGroup0;
    w[(long)p * kInvK + k] = src >= 0 ? inv[(long)src * kFilter + kHop * (3 - sh) + p] * kInvBasisScale : 0.f;
  }
}

// get_window('hann', 1024, fftbins=True) ** 2 in double (audio_processing.py:47-49)
__global__ void build_wsq_kernel(double* wsq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kFilter) {
    const double w = 0.5 - 0.5 * cos(2.0 * 3.14159265358979323846 * i / kFilter);
    wsq[i] = w * w;
  }
}

// Where row b of a window [s0, s0 + n) ends, relative to the window: closed (the sequence ends at e <= n) or open (it
// goes on past the window).  lengths[b] in [0, n] ends the row there; a negative or larger value, or no lengths, means
// the window's end: the sequence's end when at_end, else open.
struct RowEnd { bool closed; int e; };
__device__ __forceinline__ RowEnd row_end(const int32_t* len, int b, int n, int at_end) {
  const int l = len ? len[b] : -1;
  if (l >= 0 && l <= n) return RowEnd{true, l};
  return RowEnd{at_end != 0, n};
}

// 1 + the number of frames of row b (frames f with f + 1 < fend exist); 0 for a row too short to reflect-pad
__device__ __forceinline__ int frame_end(RowEnd r, int s0, int F) {
  if (!r.closed) return F + 1;
  if (s0 + r.e <= kFilter / 2) return 0;
  return min(r.e / kHop + 2, F + 1);
}

// audio (B, n) -> padded block planes: plane row 1 + b * span + i holds the padded samples 256 i ... 256 i + 255, i.e.
// the window samples u = 256 i + c - 512, reflected at the sequence's start (s0 = 0) and at a closed row's end.
// Samples no output needs (outside the window, or of a row too short to pad) are zero.  Every plane row is written.
// scale (or NULL): the samples of row b are packed times scale[b].
__global__ void pack_kernel(const void* __restrict__ audio, int io_half, int B, int n, const int32_t* __restrict__ len,
                            int at_end, int s0, int F, int span, __half* __restrict__ planes, long rows,
                            int32_t* __restrict__ fend, const float* __restrict__ scale) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y;
  if (blockIdx.x == 0 && g == 0)
    for (int b = threadIdx.x; b < B; b += blockDim.x) fend[b] = frame_end(row_end(len, b, n, at_end), s0, F);
  if (row >= rows) return;
  const long q = row - 1;
  int b = -1, i = 0;
  if (q >= 0) { b = (int)(q / span); i = (int)(q - (long)b * span); }
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = 0.f;
  if (b >= 0 && b < B && i < F + 3) {
    const RowEnd r = row_end(len, b, n, at_end);
    const int lim = r.closed ? r.e : n;
    const float sc = scale ? scale[b] : 1.f;
    if (!(r.closed && s0 + r.e <= kFilter / 2)) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        int u = kHop * i + g * 8 + k - kFilter / 2;
        if (u < 0) u = s0 == 0 ? -u : -1;
        else if (u >= lim) u = r.closed ? 2 * r.e - 2 - u : -1;
        if (u >= 0 && u < lim) {
          const long idx = (long)b * n + u;
          v[k] = (io_half ? __half2float(reinterpret_cast<const __half*>(audio)[idx]) : reinterpret_cast<const float*>(audio)[idx]) * sc;
        }
      }
    }
  }
  store8<kPassesFp32>(planes, rows, g, row, v);
}

// bias_spec: the magnitude of frame 0 of audio (n > 512 samples), reflect-padded, against the forward basis
// (stft.py:69-94, denoiser.py:36); one block per bin, summed in a fixed order
__global__ void bias_kernel(const float* __restrict__ fwd, const float* __restrict__ audio, float* __restrict__ out) {
  __shared__ float red[2][8];
  const int bin = blockIdx.x;
  float re = 0.f, im = 0.f;
  for (int k = threadIdx.x; k < kFilter; k += blockDim.x) {
    const float x = audio[abs(k - kFilter / 2)];
    re = fmaf(fwd[(long)bin * kFilter + k], x, re);
    im = fmaf(fwd[(long)(kBins + bin) * kFilter + k], x, im);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    re += __shfl_xor_sync(0xffffffffu, re, o);
    im += __shfl_xor_sync(0xffffffffu, im, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = re; red[1][threadIdx.x >> 5] = im; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.f, m = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { r += red[0][w]; m += red[1][w]; }
    out[bin] = sqrtf(__fadd_rn(__fmul_rn(r, r), __fmul_rn(m, m)));
  }
}

struct DnLayout { __half* blk; __half* spec; long rows; int32_t* fend; };
struct DnDims { int F, span, ntm; };
DnDims dn_dims(int B, int n) {
  DnDims d;
  d.F = n / kHop + 1;
  d.span = d.F + 4;
  d.ntm = (int)(((long)B * d.span + kTile - 1) / kTile);
  return d;
}
// rows: the tiles, the forward's row shifts up to +2 past the last (after its one leading row) and the inverse's up to +3
void dn_layout(Carve& c, int B, int n, DnLayout* o) {
  const DnDims d = dn_dims(B, n);
  o->rows = (long)d.ntm * kTile + 4;
  o->blk = c.take<__half>((size_t)kBlkGroups * 2 * o->rows * 8, 1024);
  o->spec = c.take<__half>((size_t)kSpecGroups * 2 * o->rows * 8, 1024);
  o->fend = c.take<int32_t>((size_t)B, 256);
}

// The STFT entry points' workspace: the denoiser's, the per-row scales, each row's length in samples (Griffin-Lim's
// packs read it) and, for Griffin-Lim, the fp32 signal (B, n) between iterations.
struct StLayout { DnLayout dn; float* scale; float* unscale; int32_t* len; float* sig; };
void st_layout(Carve& c, int B, int n, bool signal, StLayout* o) {
  dn_layout(c, B, n, &o->dn);
  o->scale = c.take<float>((size_t)B, 256);
  o->unscale = c.take<float>((size_t)B, 256);
  o->len = c.take<int32_t>((size_t)B, 256);
  o->sig = signal ? c.take<float>((size_t)B * n, 256) : nullptr;
}

// forward transform over the spectrum rows [lo, hi) of the layout (rows = frames; see the file comment)
GemmParams forward_params(const T2Denoiser* m, const DnDims& d, const DnLayout& o, int B, int lo, int hi) {
  GemmParams f;
  memset(&f, 0, sizeof(f));
  for (int j = 0; j < 4; ++j) f.seg[j] = Seg{o.blk, o.rows, j - 1, kHop / 64};
  f.nseg = 4; f.nchunks = 4 * (kHop / 64); f.row0 = 1; f.wimg = m->fwd_img; f.n_tiles_m = d.ntm;
  f.B = B; f.span = d.span; f.T = d.F + 1; f.len = o.fend; f.len_mul = 1;
  f.lo = lo; f.hi = hi;
  f.out = o.spec; f.out_rows = o.rows; f.out_row0 = 0;
  return f;
}

// inverse transform + overlap-add + envelope over the output blocks [lo, hi), written to audio (B, 256 (hi - lo))
GemmParams inverse_params(const T2Denoiser* m, const DnDims& d, const DnLayout& o, int B, int lo, int hi, float* audio) {
  GemmParams v;
  memset(&v, 0, sizeof(v));
  for (int sh = 0; sh < 4; ++sh) v.seg[sh] = Seg{o.spec, o.rows, sh, kSpecCh / 64};
  v.nseg = 4; v.nchunks = 4 * (kSpecCh / 64); v.row0 = 0; v.wimg = m->inv_img; v.n_tiles_m = d.ntm;
  v.B = B; v.span = d.span; v.T = d.F - 1; v.len = o.fend; v.len_mul = 1;
  v.lo = lo; v.hi = hi;
  v.audio = audio; v.audio_pitch = (long)kHop * (hi - lo); v.wsq = m->wsq;
  return v;
}

// ---- per-row scales: the largest |value| of a row, over the CTAs of a cluster, to a power of two -----------------
constexpr int kRowCluster = 8, kRowThreads = 512;

// max |x[r * ld + c]| over r < R, c < lim: the CTAs of the cluster take every kRowCluster-th element; every thread of
// the cluster gets the result.  Rows of the cluster's blocks are independent of every other cluster's.
__device__ float cluster_row_max(const float* __restrict__ x, int R, long ld, int lim) {
  namespace cg = cooperative_groups;
  __shared__ float red[kRowThreads / 32 + 1];
  cg::cluster_group cl = cg::this_cluster();
  const long total = (long)R * lim, stride = (long)kRowCluster * blockDim.x;
  float mx = 0.f;
  for (long i = (long)cl.block_rank() * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long r = i / lim;
    mx = fmaxf(mx, fabsf(x[r * ld + (i - r * lim)]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v = fmaxf(v, red[w]);
    red[kRowThreads / 32] = v;
  }
  cl.sync();
  float v = 0.f;
  for (int r = 0; r < kRowCluster; ++r) v = fmaxf(v, *cl.map_shared_rank(&red[kRowThreads / 32], r));
  cl.sync();                                  // no CTA leaves while a peer may still read its shared memory
  return v;
}

// 2^k with mx 2^k in [2^(top - 1), 2^top); 1 for a row of zeros (or inf / NaN)
__device__ __forceinline__ float pow2_scale(float mx, int top) {
  if (!(mx > 0.f) || isinf(mx)) return 1.f;
  int e;
  frexpf(mx, &e);
  return ldexpf(1.f, min(max(top - e, -126), 127));
}

// transform: scale[b] brings row b's largest |sample| (of its first lengths[b] samples) into [0.5, 1)
__global__ void __cluster_dims__(kRowCluster, 1, 1) __launch_bounds__(kRowThreads)
audio_scale_kernel(const float* __restrict__ audio, int n, const int32_t* __restrict__ len, float* __restrict__ scale,
                   float* __restrict__ unscale) {
  const int b = blockIdx.y;
  const float mx = cluster_row_max(audio + (long)b * n, 1, n, row_end(len, b, n, 1).e);
  if (cooperative_groups::this_cluster().block_rank() == 0 && threadIdx.x == 0) {
    const float s = pow2_scale(mx, 0);
    scale[b] = s;
    unscale[b] = 1.f / s;
  }
}

// inverse / Griffin-Lim input: (magnitude, phase) (B, 513, F) fp32 -> the spectrum planes the inverse GEMM reads,
// (m cos phase, m sin phase) scale[b] / 512 at plane row b * span + 1 + f, zeros in the other rows of the sequence.
// Row b has Fb = frames[b] frames (F for NULL or a value outside [0, F]); a row of fewer than 4 frames (at most 512
// samples) cannot be reflect-padded by its transforms and gives zeros.  scale[b] brings the row's largest magnitude to
// [512, 1024), the range of the spectrum of unit-scale audio.  Also writes unscale = 1 / scale, the row's length in
// samples, 256 (Fb - 1), and fend as pack_kernel computes it from that length.  One cluster per row.
__global__ void __cluster_dims__(kRowCluster, 1, 1) __launch_bounds__(kRowThreads)
spec_pack_kernel(const float* __restrict__ mag, const float* __restrict__ phase, const int32_t* __restrict__ frames,
                 int F, int span, __half* __restrict__ planes, long rows, float* __restrict__ scale,
                 float* __restrict__ unscale, int32_t* __restrict__ len, int32_t* __restrict__ fend) {
  const int b = blockIdx.y, rank = (int)cooperative_groups::this_cluster().block_rank();
  const int l = frames ? frames[b] : -1;
  const int Fb = l >= 0 && l <= F ? l : F;
  const int fe = Fb >= 4 ? Fb + 1 : 0;
  const float* mb = mag + (long)b * kBins * F;
  const float* pb = phase + (long)b * kBins * F;
  const float s = pow2_scale(cluster_row_max(mb, kBins, F, fe ? Fb : 0), 10), sc = s * kSpecScale;
  if (rank == 0 && threadIdx.x == 0) {
    scale[b] = s;
    unscale[b] = 1.f / s;
    len[b] = fe ? kHop * (Fb - 1) : 0;
    fend[b] = fe;
  }
  // item (j, t): j < 65 is bins 8 j ... 8 j + 7 of row t (real parts to group j, imaginary to group 65 + j); j in
  // [65, 71) zeroes group 65 + j, the padding groups 130 ... 135
  const int items = (kSpecGroups - kImGroup0) * span;
  for (int it = rank * blockDim.x + threadIdx.x; it < items; it += kRowCluster * blockDim.x) {
    const int j = it / span, t = it - j * span;
    const long q = (long)b * span + t;
    float re[8], im[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int bin = 8 * j + i;
      re[i] = im[i] = 0.f;
      if (j < kImGroup0 && bin < kBins && t >= 1 && t < fe) {
        const float m = mb[(long)bin * F + t - 1], ph = pb[(long)bin * F + t - 1];
        re[i] = __fmul_rn(m, cosf(ph)) * sc;
        im[i] = __fmul_rn(m, sinf(ph)) * sc;
      }
    }
    if (j < kImGroup0) store8<kPassesFp32>(planes, rows, j, q, re);
    store8<kPassesFp32>(planes, rows, kImGroup0 + j, q, im);
  }
}

}  // namespace

static int pack(T2Denoiser* m, const float* fwd, const float* inv, cudaStream_t s) {
  T2_CUDA(cudaMemcpyAsync(m->fwd, fwd, (size_t)kBasisRows * kFilter * sizeof(float), cudaMemcpyDeviceToDevice, s));
  build_fwd_kernel<<<kFwdN, 256, 0, s>>>(fwd, m->tmp);
  T2_LAUNCH_CHECK();
  T2_TRY(tc_pack_weights(m->tmp, kFwdN, kFilter, 1, kNT, &m->fwd_img, s));
  build_inv_kernel<<<kHop, 256, 0, s>>>(inv, m->tmp);
  T2_LAUNCH_CHECK();
  T2_TRY(tc_pack_weights(m->tmp, kHop, kInvK, 1, kNT, &m->inv_img, s));
  return T2_OK;
}

int denoiser_create(T2Denoiser** out, const T2DenoiserConfig* c, const float* fwd, const float* inv, cudaStream_t s) {
  if (!out || !c || !fwd || !inv) return fail(T2_ERR_INVALID, "denoiser: null argument");
  if (c->filter_length != kFilter || c->hop_length != kHop || c->win_length != kFilter || c->window != T2_WINDOW_HANN)
    return fail(T2_ERR_UNSUPPORTED, "denoiser: the sm_90a kernels are built for filter_length 1024, hop 256, win_length "
                                     "1024 and a Hann window (got %d / %d / %d, window %d)",
                c->filter_length, c->hop_length, c->win_length, c->window);
  int dev = 0;
  T2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  T2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) return fail(T2_ERR_UNSUPPORTED, "libt2b200 is built for sm_90a only (device is sm_%d%d)", p.major, p.minor);
  T2Denoiser* m = new T2Denoiser();
  int r = T2_OK;
  if (cudaMalloc((void**)&m->fwd, (size_t)kBasisRows * kFilter * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&m->wsq, kFilter * sizeof(double)) != cudaSuccess ||
      cudaMalloc((void**)&m->tmp, (size_t)std::max(kFwdN * kFilter, kHop * kInvK) * sizeof(float)) != cudaSuccess)
    r = fail(T2_ERR_CUDA, "denoiser: out of device memory for the packed bases");
  if (r == T2_OK) {
    build_wsq_kernel<<<kFilter / 256, 256, 0, s>>>(m->wsq);
    if (cudaGetLastError() != cudaSuccess) r = fail(T2_ERR_CUDA, "denoiser: window kernel launch failed");
    else g_launch_count++;
  }
  if (r == T2_OK) r = pack(m, fwd, inv, s);
  if (r != T2_OK) { denoiser_destroy(m); return r; }
  *out = m;
  return T2_OK;
}

int denoiser_refresh(T2Denoiser* m, const float* fwd, const float* inv, cudaStream_t s) {
  if (!m || !fwd || !inv) return fail(T2_ERR_INVALID, "denoiser: null argument");
  return pack(m, fwd, inv, s);
}

int denoiser_destroy(T2Denoiser* m) {
  if (!m) return T2_OK;
  cudaFree(m->fwd); cudaFree(m->fwd_img); cudaFree(m->inv_img); cudaFree(m->wsq); cudaFree(m->tmp);
  delete m;
  return T2_OK;
}

int denoiser_bias(T2Denoiser* m, const float* audio, int n, float* bias_out, cudaStream_t s) {
  if (!m || !audio || !bias_out) return fail(T2_ERR_INVALID, "denoiser: null argument");
  if (n <= kFilter / 2) return fail(T2_ERR_INVALID, "denoiser bias: %d samples cannot be reflect-padded by 512", n);
  bias_kernel<<<kBins, 256, 0, s>>>(m->fwd, audio, bias_out);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

size_t denoiser_ws_bytes(int B, int n) {
  Carve c(nullptr, 1024);
  DnLayout o;
  dn_layout(c, B, n, &o);
  return c.bytes();
}

void denoiser_window_halo(int* left, int* right) {
  if (left) *left = kHalo;
  if (right) *right = kHalo;
}

int denoiser_run(T2Denoiser* m, const T2DenoiserArgs* a, cudaStream_t s) {
  if (!a) return fail(T2_ERR_INVALID, "denoiser: null argument");
  if (a->lengths && a->n > 0 && a->n < kHop) return T2_OK;       // no output block (every row is too short)
  T2DenoiserWindowArgs w;
  memset(&w, 0, sizeof(w));
  w.dn = *a;
  w.s0 = 0; w.out0 = 0; w.out1 = a->n / kHop; w.at_end = 1;
  return denoiser_run_window(m, &w, s);
}

int denoiser_run_window(T2Denoiser* m, const T2DenoiserWindowArgs* wa, cudaStream_t s) {
  if (!m || !wa || !wa->dn.audio || !wa->dn.bias || !wa->dn.out || !wa->dn.ws) return fail(T2_ERR_INVALID, "denoiser: null argument");
  const T2DenoiserArgs* a = &wa->dn;
  const int B = a->B, n = a->n, s0 = wa->s0, out0 = wa->out0, out1 = wa->out1;
  if (B <= 0 || n <= 0) return fail(T2_ERR_INVALID, "denoiser: empty input (B=%d, n=%d)", B, n);
  if ((long)B * (n / kHop + 5) > (1L << 30) || (long)s0 + n > (1L << 31) - 1)
    return fail(T2_ERR_INVALID, "denoiser: input too large");
  if (s0 < 0 || s0 % kHop) return fail(T2_ERR_INVALID, "denoiser window: s0 = %d is not a non-negative multiple of 256", s0);
  if (!a->lengths && wa->at_end && s0 + n <= kFilter / 2)
    return fail(T2_ERR_INVALID, "denoiser: %d samples cannot be reflect-padded by 512", s0 + n);
  if (out0 < 0 || out1 <= out0 || out1 > n / kHop)
    return fail(T2_ERR_INVALID, "denoiser window: output blocks [%d, %d) are not a non-empty range of the window's %d "
                "blocks", out0, out1, n / kHop);
  if (s0 > 0 && out0 < kHalo)
    return fail(T2_ERR_INVALID, "denoiser window: output starts %d blocks after a window start that is not the "
                "sequence's start; the left halo is %d blocks", out0, kHalo);
  if (!wa->at_end && out1 + kHalo > n / kHop)
    return fail(T2_ERR_INVALID, "denoiser window: output ends %d blocks before a window end that is not the sequence's "
                "end; the right halo is %d blocks", n / kHop - out1, kHalo);
  if (reinterpret_cast<uintptr_t>(a->out) % 16)
    return fail(T2_ERR_INVALID, "denoiser: out must be 16-byte aligned (the epilogue writes it with 16-byte stores)");
  if (a->ws_bytes < denoiser_ws_bytes(B, n)) return fail(T2_ERR_WORKSPACE, "denoiser workspace too small");
  const DnDims d = dn_dims(B, n);
  Carve c(a->ws, 1024);
  DnLayout o;
  dn_layout(c, B, n, &o);
  pack_kernel<<<dim3((unsigned)((o.rows + 127) / 128), kBlkGroups), 128, 0, s>>>(
      a->audio, a->io_half, B, n, a->lengths, wa->at_end, s0, d.F, d.span, o.blk, o.rows, o.fend, nullptr);
  T2_LAUNCH_CHECK();
  // forward transform + spectral gate over the spectrum rows the output blocks read: [out0, out1 + 3)
  GemmParams f = forward_params(m, d, o, B, out0, std::min(d.span, out1 + kHalo));
  f.bias = a->bias; f.strength = a->strength;
  T2_TRY((launch_gemm<EPI_SPECTRAL, kPassesFp32>(f, kFwdTiles, s)));
  // inverse transform + overlap-add + envelope over the output blocks [out0, out1)
  T2_TRY((launch_gemm<EPI_OVERLAP, kPassesFp32>(inverse_params(m, d, o, B, out0, out1, a->out), 1, s)));
  return T2_OK;
}

// ---- public STFT transform / inverse and Griffin-Lim ----------------------------------------------------------------
// Checks shared by the entry points that take a (B, 513, F) spectrum; F >= 4 frames make 256 (F - 1) > 512 samples,
// which the reference's reflect padding needs.
static int check_spectrum(const char* what, T2Denoiser* m, const T2StftInverseArgs* a, bool signal) {
  if (!m || !a || !a->magnitude || !a->phase || !a->out || !a->ws) return fail(T2_ERR_INVALID, "%s: null argument", what);
  if (a->B <= 0) return fail(T2_ERR_INVALID, "%s: empty batch (B=%d)", what, a->B);
  if (a->F < 4)
    return fail(T2_ERR_INVALID, "%s: %d frames give %d samples, which cannot be reflect-padded by 512 (at least 4 "
                "frames are needed)", what, a->F, kHop * (a->F - 1));
  if ((long)a->B * (a->F + 4) > (1L << 30) || (long)kHop * (a->F - 1) > (1L << 31) - 1)
    return fail(T2_ERR_INVALID, "%s: input too large", what);
  if (reinterpret_cast<uintptr_t>(a->out) % 16)
    return fail(T2_ERR_INVALID, "%s: out must be 16-byte aligned (the epilogue writes it with 16-byte stores)", what);
  if (a->ws_bytes < stft_ws_bytes(a->B, kHop * (a->F - 1), signal)) return fail(T2_ERR_WORKSPACE, "%s workspace too small", what);
  return T2_OK;
}

size_t stft_ws_bytes(int B, int n, bool signal) {
  Carve c(nullptr, 1024);
  StLayout o;
  st_layout(c, B, n, signal, &o);
  return c.bytes();
}

int stft_transform(T2Denoiser* m, const T2StftTransformArgs* a, cudaStream_t s) {
  if (!m || !a || !a->audio || !a->magnitude || !a->phase || !a->ws) return fail(T2_ERR_INVALID, "stft transform: null argument");
  const int B = a->B, n = a->n;
  if (B <= 0 || n <= 0) return fail(T2_ERR_INVALID, "stft transform: empty input (B=%d, n=%d)", B, n);
  if ((long)B * (n / kHop + 5) > (1L << 30)) return fail(T2_ERR_INVALID, "stft transform: input too large");
  if (!a->lengths && n <= kFilter / 2)
    return fail(T2_ERR_INVALID, "stft transform: %d samples cannot be reflect-padded by 512", n);
  if (a->ws_bytes < stft_ws_bytes(B, n, false)) return fail(T2_ERR_WORKSPACE, "stft transform workspace too small");
  const DnDims d = dn_dims(B, n);
  Carve c(a->ws, 1024);
  StLayout o;
  st_layout(c, B, n, false, &o);
  audio_scale_kernel<<<dim3(kRowCluster, B), kRowThreads, 0, s>>>(a->audio, n, a->lengths, o.scale, o.unscale);
  T2_LAUNCH_CHECK();
  pack_kernel<<<dim3((unsigned)((o.dn.rows + 127) / 128), kBlkGroups), 128, 0, s>>>(
      a->audio, 0, B, n, a->lengths, 1, 0, d.F, d.span, o.dn.blk, o.dn.rows, o.dn.fend, o.scale);
  T2_LAUNCH_CHECK();
  GemmParams f = forward_params(m, d, o.dn, B, 0, d.F + 1);
  f.row_scale = o.unscale; f.mag_out = a->magnitude; f.phase_out = a->phase;
  T2_TRY((launch_gemm<EPI_MAGPHASE, kPassesFp32>(f, kFwdTiles, s)));
  return T2_OK;
}

// spectrum planes from (magnitude, phase), then the inverse into out (times unscale: the caller's units) or, with
// unscale NULL, into the scaled signal Griffin-Lim iterates on
static int spec_pack(const T2StftInverseArgs* a, const DnDims& d, const StLayout& o, cudaStream_t s) {
  spec_pack_kernel<<<dim3(kRowCluster, a->B), kRowThreads, 0, s>>>(a->magnitude, a->phase, a->lengths, d.F, d.span,
                                                                  o.dn.spec, o.dn.rows, o.scale, o.unscale, o.len,
                                                                  o.dn.fend);
  T2_LAUNCH_CHECK();
  return T2_OK;
}
static int inverse_to(T2Denoiser* m, int B, const DnDims& d, const StLayout& o, float* out, const float* unscale,
                      cudaStream_t s) {
  GemmParams v = inverse_params(m, d, o.dn, B, 0, d.F - 1, out);
  v.row_scale = unscale;
  return launch_gemm<EPI_OVERLAP, kPassesFp32>(v, 1, s);
}

int stft_inverse(T2Denoiser* m, const T2StftInverseArgs* a, cudaStream_t s) {
  T2_TRY(check_spectrum("stft inverse", m, a, false));
  const int B = a->B, n = kHop * (a->F - 1);
  const DnDims d = dn_dims(B, n);
  Carve c(a->ws, 1024);
  StLayout o;
  st_layout(c, B, n, false, &o);
  T2_TRY(spec_pack(a, d, o, s));
  return inverse_to(m, B, d, o, a->out, o.unscale, s);
}

int griffin_lim(T2Denoiser* m, const T2GriffinLimArgs* g, cudaStream_t s) {
  if (!g) return fail(T2_ERR_INVALID, "griffin_lim: null argument");
  const T2StftInverseArgs* a = &g->inv;
  T2_TRY(check_spectrum("griffin_lim", m, a, true));
  if (g->n_iters < 0) return fail(T2_ERR_INVALID, "griffin_lim: n_iters = %d is negative", g->n_iters);
  const int B = a->B, n = kHop * (a->F - 1);
  const DnDims d = dn_dims(B, n);
  Carve c(a->ws, 1024);
  StLayout o;
  st_layout(c, B, n, true, &o);
  // signal = inverse(S, angles); then n_iters times: signal = inverse(S, phase of transform(signal))
  T2_TRY(spec_pack(a, d, o, s));
  T2_TRY(inverse_to(m, B, d, o, g->n_iters == 0 ? a->out : o.sig, g->n_iters == 0 ? o.unscale : nullptr, s));
  for (int i = 1; i <= g->n_iters; ++i) {
    pack_kernel<<<dim3((unsigned)((o.dn.rows + 127) / 128), kBlkGroups), 128, 0, s>>>(
        o.sig, 0, B, n, o.len, 1, 0, d.F, d.span, o.dn.blk, o.dn.rows, o.dn.fend, nullptr);
    T2_LAUNCH_CHECK();
    GemmParams f = forward_params(m, d, o.dn, B, 0, std::min(d.span, d.F - 1 + kHalo));
    f.target = a->magnitude; f.row_scale = o.scale;
    T2_TRY((launch_gemm<EPI_PROJECT, kPassesFp32>(f, kFwdTiles, s)));
    const bool last = i == g->n_iters;
    T2_TRY(inverse_to(m, B, d, o, last ? a->out : o.sig, last ? o.unscale : nullptr, s));
  }
  return T2_OK;
}

}  // namespace t2
