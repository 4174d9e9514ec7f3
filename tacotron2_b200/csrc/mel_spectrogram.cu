// GPU log-mel extraction: TacotronSTFT.mel_spectrogram (layers.py:63-80, stft.py:69-94; SURVEY.md section 8(f) item 4).
//
//   y (B, n) in [-1, 1]  -> reflect-pad by filter_length / 2 on both sides                        (stft.py:76-81)
//                        -> frames x windowed Fourier basis: ONE strided-batch tensor-core GEMM     (stft.py:83-87)
//                             A[b] = the padded signal of row b read with leading dimension hop_length: frame f is
//                             y_pad[f * hop : f * hop + filter_length] -- overlapping rows, nothing is materialised
//                             B    = forward_basis (2 * cutoff, filter_length), shared by the batch
//                        -> magnitude sqrt(re^2 + im^2)                                             (stft.py:89-91)
//                        -> mel_basis (n_mel, cutoff) x magnitudes: second GEMM                     (layers.py:78)
//                        -> log(clamp(., clip_val)), written as (B, n_mel, n_frames)                (layers.py:79, audio_processing.py:78-84)
//
// Both products run on gemm_tc.cu (split-fp16 wgmma, fp32-grade).  Without lengths a batch shares each frame's operand
// scale (the maximum over the batch) and plans its K splits for the whole batch, so a row's bits depend on the rows it is
// batched with; that call is kept as it is.  With lengths (T2MelSpecArgs.lengths) every row is computed as its own B = 1
// call: padded at its own end, and both products use gemm_tc's ragged entries (per-row scales, the B = 1 K-split plan).
#include <algorithm>

#include "gemm_tc.h"

namespace t2 {
namespace {

// lengths (device, per row, or nullptr = n for every row): row b is y[b, :n_b] padded at its own end, and the rest of its
// n + 2 pad slots is zeroed; block (0, b) also writes the row's frame count n_b / hop + 1.  Lengths are clamped to
// [pad + 1, n] (the caller refuses others) so that nothing outside the row is ever read.
__device__ __forceinline__ int row_length(const int* __restrict__ lengths, int b, int n, int pad) {
  return lengths ? min(max(lengths[b], pad + 1), n) : n;
}
__global__ void reflect_pad_kernel(const float* __restrict__ y, int n, int pad, const int* __restrict__ lengths, int hop,
                                   int* __restrict__ frames, float* __restrict__ out) {
  const long row = (long)n + 2 * pad;
  const int nb = row_length(lengths, blockIdx.y, n, pad);
  const long total = (long)nb + 2 * pad;
  const float* src = y + (long)blockIdx.y * n;
  float* dst = out + (long)blockIdx.y * row;
  if (lengths && blockIdx.x == 0 && threadIdx.x == 0) frames[blockIdx.y] = nb / hop + 1;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < row; i += (long)gridDim.x * blockDim.x) {
    if (i >= total) { dst[i] = 0.f; continue; }
    long j = i - pad;                       // F.pad(mode='reflect'): the edge sample is not repeated
    if (j < 0) j = -j;
    if (j >= nb) j = 2L * (nb - 1) - j;
    dst[i] = src[j];
  }
}
// frames (device, per row, or nullptr): rows f >= frames[b] of batch entry b (n_frames rows each) are skipped
__global__ void magnitude_kernel(const float* __restrict__ ft, long rows, int cutoff, const int* __restrict__ frames,
                                 int n_frames, float* __restrict__ mag) {
  const long total = rows * cutoff;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / cutoff;
    const int c = (int)(i - r * cutoff);
    if (frames && r % n_frames >= frames[r / n_frames]) continue;
    const float re = ft[r * 2 * cutoff + c], im = ft[r * 2 * cutoff + cutoff + c];
    mag[i] = sqrtf(re * re + im * im);
  }
}
// mel (B * n_frames, n_mel) -> out (B, n_mel, n_frames) = log(max(mel, clip)); frames (device, per row, or nullptr):
// frames f >= frames[b] of row b are written as zeros and their mel values are not read
__global__ void log_transpose_kernel(const float* __restrict__ mel, int n_frames, int n_mel, float clip,
                                     const int* __restrict__ frames, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, f0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  const int fb = frames ? frames[b] : n_frames;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int f = f0 + r, mm = m0 + threadIdx.x;
    tile[r][threadIdx.x] = (f < fb && mm < n_mel) ? mel[((long)b * n_frames + f) * n_mel + mm] : 1.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int mm = m0 + r, f = f0 + threadIdx.x;
    if (mm < n_mel && f < n_frames) out[((long)b * n_mel + mm) * n_frames + f] = f < fb ? logf(fmaxf(tile[threadIdx.x][r], clip)) : 0.f;
  }
}

// ragged (per-row lengths): both products take gemm_tc's ragged entries, whose scratch replaces the unlengthed one's,
// and the frame count of every row follows
struct MelSpecWs { float *ypad, *ft, *mag, *mel; void* gemm; size_t gemm_bytes; int* frames; };
void mel_ws_layout(Carve& c, int B, int n, int fl, int hop, int n_mel, bool ragged, MelSpecWs* w) {
  const long frames = n / hop + 1, cutoff = fl / 2 + 1;
  w->ypad = c.take<float>((size_t)B * (n + fl));                // reflect-padded signal
  w->ft = c.take<float>((size_t)B * frames * 2 * cutoff);       // Fourier transform (real | imaginary)
  w->mag = c.take<float>((size_t)B * frames * cutoff);
  w->mel = c.take<float>((size_t)B * frames * n_mel);           // (B frames, n_mel) before the log / transpose
  if (ragged)
    w->gemm_bytes = std::max(gemm_tc_ragged_ws_bytes((int)frames, (int)(2 * cutoff), B),
                             gemm_tc_ragged_ws_bytes((int)frames, n_mel, B));
  else
    w->gemm_bytes = std::max(gemm_tc_ws_bytes((int)frames, (int)(2 * cutoff), fl, B),
                             gemm_tc_ws_bytes((int)(B * frames), n_mel, (int)cutoff));
  w->gemm = c.take<char>(w->gemm_bytes);                        // scratch of both products
  w->frames = ragged ? c.take<int>((size_t)B) : nullptr;        // frames of each row
}

}  // namespace
}  // namespace t2

extern "C" {

int32_t t2_mel_spectrogram_frames(int32_t n_samples, int32_t hop_length) { return n_samples / hop_length + 1; }

static size_t mel_ws_bytes(int B, int n, int fl, int hop, int n_mel, bool ragged) {
  using namespace t2;
  Carve c(nullptr);
  MelSpecWs w;
  mel_ws_layout(c, B, n, fl, hop, n_mel, ragged, &w);
  return c.bytes();
}
size_t t2_mel_spectrogram_workspace_bytes(int32_t B, int32_t n_samples, int32_t filter_length, int32_t hop_length, int32_t n_mel) {
  return mel_ws_bytes(B, n_samples, filter_length, hop_length, n_mel, false);
}
size_t t2_mel_spectrogram_workspace_bytes_lengths(int32_t B, int32_t n_max, int32_t filter_length, int32_t hop_length,
                                                  int32_t n_mel) {
  return mel_ws_bytes(B, n_max, filter_length, hop_length, n_mel, true);
}

int t2_mel_spectrogram(const T2MelSpecArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->y || !a->forward_basis || !a->mel_basis || !a->mel || !a->ws) return fail(T2_ERR_INVALID, "mel_spectrogram: null argument");
  const int B = a->B, n = a->n_samples, fl = a->filter_length, hop = a->hop_length, n_mel = a->n_mel;
  if (B <= 0 || n <= 0 || fl <= 0 || (fl & 1) || hop <= 0 || n_mel <= 0)
    return fail(T2_ERR_INVALID, "mel_spectrogram: bad sizes (B %d, n_samples %d, filter_length %d, hop_length %d, n_mel %d)",
                B, n, fl, hop, n_mel);
  if (n <= fl / 2) return fail(T2_ERR_INVALID, "mel_spectrogram: reflect padding needs n_samples > filter_length / 2 (got %d)", n);
  const bool ragged = a->lengths != nullptr;
  if (a->ws_bytes < mel_ws_bytes(B, n, fl, hop, n_mel, ragged)) return fail(T2_ERR_WORKSPACE, "mel_spectrogram workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  const int frames = n / hop + 1, cutoff = fl / 2 + 1;
  const long padded = (long)n + fl;
  Carve c(a->ws);
  MelSpecWs w;
  mel_ws_layout(c, B, n, fl, hop, n_mel, ragged, &w);
  reflect_pad_kernel<<<dim3((unsigned)((padded + 255) / 256 > 1024 ? 1024 : (padded + 255) / 256), B), 256, 0, s>>>(
      a->y, n, fl / 2, a->lengths, hop, w.frames, w.ypad);
  T2_LAUNCH_CHECK();
  GemmTc g;                                   // w.ft[b] (frames x 2 cutoff) = frames(b) . forward_basis^T
  g.ta = false; g.tb = true; g.M = frames; g.N = 2 * cutoff; g.K = fl;
  g.A = w.ypad; g.lda = hop; g.strideA = padded;
  g.B = a->forward_basis; g.ldb = fl; g.strideB = 0;
  g.C = w.ft; g.ldc = 2 * cutoff; g.strideC = (long)frames * 2 * cutoff; g.batch = B;
  g.ws = w.gemm; g.ws_bytes = w.gemm_bytes;
  g.entry_rows = w.frames;                    // ragged: each row as its own B = 1 product
  T2_TRY(gemm_tc(kGemmTcSms, s, g));
  const long rows = (long)B * frames;
  magnitude_kernel<<<(unsigned)((rows * cutoff + 255) / 256 > 4096 ? 4096 : (rows * cutoff + 255) / 256), 256, 0, s>>>(
      w.ft, rows, cutoff, w.frames, frames, w.mag);
  T2_LAUNCH_CHECK();
  if (ragged) {                               // w.mel[b] (frames x n_mel) = mag(b) . mel_basis^T, planned per row
    GemmTc m;
    m.ta = false; m.tb = true; m.M = frames; m.N = n_mel; m.K = cutoff;
    m.A = w.mag; m.lda = cutoff; m.strideA = (long)frames * cutoff;
    m.B = a->mel_basis; m.ldb = cutoff; m.strideB = 0;
    m.C = w.mel; m.ldc = n_mel; m.strideC = (long)frames * n_mel; m.batch = B;
    m.ws = w.gemm; m.ws_bytes = w.gemm_bytes; m.entry_rows = w.frames;
    T2_TRY(gemm_tc(kGemmTcSms, s, m));
  } else {
    T2_TRY(gemm_tc_rm(kGemmTcSms, s, w.gemm, w.gemm_bytes, false, true, (int)rows, n_mel, cutoff, w.mag, cutoff, a->mel_basis,
                      cutoff, w.mel, n_mel, 0.f));
  }
  log_transpose_kernel<<<dim3((frames + 31) / 32, (n_mel + 31) / 32, B), dim3(32, 8), 0, s>>>(w.mel, frames, n_mel, a->clip_val,
                                                                                             w.frames, a->mel);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
