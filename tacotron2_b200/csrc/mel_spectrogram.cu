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
// Both products run on gemm_tc.cu (split-fp16 wgmma, fp32-grade).
#include "gemm_tc.h"

namespace t2 {
namespace {

__global__ void reflect_pad_kernel(const float* __restrict__ y, int n, int pad, float* __restrict__ out) {
  const long total = (long)n + 2 * pad;
  const float* src = y + (long)blockIdx.y * n;
  float* dst = out + (long)blockIdx.y * total;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    long j = i - pad;                       // F.pad(mode='reflect'): the edge sample is not repeated
    if (j < 0) j = -j;
    if (j >= n) j = 2L * (n - 1) - j;
    dst[i] = src[j];
  }
}
__global__ void magnitude_kernel(const float* __restrict__ ft, long rows, int cutoff, float* __restrict__ mag) {
  const long total = rows * cutoff;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / cutoff;
    const int c = (int)(i - r * cutoff);
    const float re = ft[r * 2 * cutoff + c], im = ft[r * 2 * cutoff + cutoff + c];
    mag[i] = sqrtf(re * re + im * im);
  }
}
// mel (B * n_frames, n_mel) -> out (B, n_mel, n_frames) = log(max(mel, clip))
__global__ void log_transpose_kernel(const float* __restrict__ mel, int n_frames, int n_mel, float clip, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, f0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int f = f0 + r, mm = m0 + threadIdx.x;
    tile[r][threadIdx.x] = (f < n_frames && mm < n_mel) ? mel[((long)b * n_frames + f) * n_mel + mm] : 1.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int mm = m0 + r, f = f0 + threadIdx.x;
    if (mm < n_mel && f < n_frames) out[((long)b * n_mel + mm) * n_frames + f] = logf(fmaxf(tile[threadIdx.x][r], clip));
  }
}

struct MelSpecWs { float *ypad, *ft, *mag, *mel; };
void mel_ws_layout(Carve& c, int B, int n, int fl, int hop, int n_mel, MelSpecWs* w) {
  const long frames = n / hop + 1, cutoff = fl / 2 + 1;
  w->ypad = c.take<float>((size_t)B * (n + fl));                // reflect-padded signal
  w->ft = c.take<float>((size_t)B * frames * 2 * cutoff);       // Fourier transform (real | imaginary)
  w->mag = c.take<float>((size_t)B * frames * cutoff);
  w->mel = c.take<float>((size_t)B * frames * n_mel);           // (B frames, n_mel) before the log / transpose
}

}  // namespace
}  // namespace t2

extern "C" {

int32_t t2_mel_spectrogram_frames(int32_t n_samples, int32_t hop_length) { return n_samples / hop_length + 1; }

size_t t2_mel_spectrogram_workspace_bytes(int32_t B, int32_t n_samples, int32_t filter_length, int32_t hop_length, int32_t n_mel) {
  using namespace t2;
  Carve c(nullptr);
  MelSpecWs w;
  mel_ws_layout(c, B, n_samples, filter_length, hop_length, n_mel, &w);
  return c.bytes();
}

int t2_mel_spectrogram(const T2MelSpecArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->y || !a->forward_basis || !a->mel_basis || !a->mel || !a->ws) return fail(T2_ERR_INVALID, "mel_spectrogram: null argument");
  const int B = a->B, n = a->n_samples, fl = a->filter_length, hop = a->hop_length, n_mel = a->n_mel;
  if (B <= 0 || n <= 0 || fl <= 0 || (fl & 1) || hop <= 0 || n_mel <= 0) return fail(T2_ERR_INVALID, "mel_spectrogram: bad sizes");
  if (n <= fl / 2) return fail(T2_ERR_INVALID, "mel_spectrogram: reflect padding needs n_samples > filter_length / 2 (got %d)", n);
  if (a->ws_bytes < t2_mel_spectrogram_workspace_bytes(B, n, fl, hop, n_mel)) return fail(T2_ERR_WORKSPACE, "mel_spectrogram workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  const int frames = n / hop + 1, cutoff = fl / 2 + 1;
  const long padded = (long)n + fl;
  Carve c(a->ws);
  MelSpecWs w;
  mel_ws_layout(c, B, n, fl, hop, n_mel, &w);
  static T2Model scratch_owner;               // only its GEMM scratch is used (grown on demand, kept for the process)
  reflect_pad_kernel<<<dim3((unsigned)((padded + 255) / 256 > 1024 ? 1024 : (padded + 255) / 256), B), 256, 0, s>>>(a->y, n, fl / 2, w.ypad);
  T2_LAUNCH_CHECK();
  GemmTc g;                                   // w.ft[b] (frames x 2 cutoff) = frames(b) . forward_basis^T
  g.ta = false; g.tb = true; g.M = frames; g.N = 2 * cutoff; g.K = fl;
  g.A = w.ypad; g.lda = hop; g.strideA = padded;
  g.B = a->forward_basis; g.ldb = fl; g.strideB = 0;
  g.C = w.ft; g.ldc = 2 * cutoff; g.strideC = (long)frames * 2 * cutoff; g.batch = B;
  T2_TRY(gemm_tc(&scratch_owner, s, g));
  const long rows = (long)B * frames;
  magnitude_kernel<<<(unsigned)((rows * cutoff + 255) / 256 > 4096 ? 4096 : (rows * cutoff + 255) / 256), 256, 0, s>>>(w.ft, rows, cutoff, w.mag);
  T2_LAUNCH_CHECK();
  T2_TRY(gemm_tc_rm(&scratch_owner, s, false, true, (int)rows, n_mel, cutoff, w.mag, cutoff, a->mel_basis, cutoff, w.mel, n_mel, 0.f));
  log_transpose_kernel<<<dim3((frames + 31) / 32, (n_mel + 31) / 32, B), dim3(32, 8), 0, s>>>(w.mel, frames, n_mel, a->clip_val, a->mel);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
