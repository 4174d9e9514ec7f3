// Fused mel-side tail of the training step (SURVEY.md section 8(f) item 3): Tacotron2Loss (loss_function.py:8-19) over
// the parse_output-masked model outputs (model.py:487-497) in ONE pass that also produces the gradient seeds:
//
//     loss   = MSE(mel, target) + MSE(mel_postnet, target) + BCEWithLogits(gate, gate_target)      (means over ALL elements,
//                                                                                                    padded frames included)
//     d_mel  = 2 (mel - target) / N_mel,   d_post = 2 (mel_postnet - target) / N_mel,
//     d_gate = (sigmoid(gate) - gate_target) / N_gate
//
// and, when output_lengths is given, applies the parse_output mask on the fly (mel / mel_postnet <- 0, gate <- 1e3 for
// frames t >= output_lengths[b]) -- in place, like the reference does through .data -- so the postnet's residual-added
// output needs no separate masked_fill pass.  Block partial sums are added in double in a fixed order (bit-reproducible).
#include <math.h>

#include "common.cuh"

namespace t2 {
namespace {

constexpr int kLossSplit = 1024;

__global__ void __launch_bounds__(256) loss_part_kernel(float* __restrict__ mel, float* __restrict__ post, float* __restrict__ gate,
                                                        const float* __restrict__ mel_t, const float* __restrict__ gate_t,
                                                        const int32_t* __restrict__ lengths, int B, int C, int T,
                                                        float* __restrict__ d_mel, float* __restrict__ d_post, float* __restrict__ d_gate,
                                                        double* __restrict__ part) {
  __shared__ double red[3][8];
  const long n_mel = (long)B * C * T, n_gate = (long)B * T;
  const float k_mel = 2.f / (float)n_mel, k_gate = 1.f / (float)n_gate;
  double s_mel = 0.0, s_post = 0.0, s_gate = 0.0;
  float a_mel = 0.f, a_post = 0.f, a_gate = 0.f;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_mel; i += stride) {      // (B, C, T) contiguous
    const int t = (int)(i % T);
    const int b = (int)(i / ((long)C * T));
    float m = mel[i], p = post[i];
    if (lengths && t >= lengths[b]) {                                                        // model.py:492-493
      m = 0.f; p = 0.f;
      mel[i] = 0.f; post[i] = 0.f;
    }
    const float tg = mel_t[i];
    const float dm = m - tg, dp = p - tg;
    a_mel = fmaf(dm, dm, a_mel); a_post = fmaf(dp, dp, a_post);
    if (d_mel) d_mel[i] = k_mel * dm;
    if (d_post) d_post[i] = k_mel * dp;
  }
  s_mel = a_mel; s_post = a_post;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_gate; i += stride) {
    const int t = (int)(i % T), b = (int)(i / T);
    float x = gate[i];
    if (lengths && t >= lengths[b]) { x = 1e3f; gate[i] = x; }                               // model.py:494
    const float y = gate_t[i];
    // BCEWithLogits: max(x, 0) - x y + log(1 + exp(-|x|))
    a_gate += fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
    if (d_gate) d_gate[i] = k_gate * (1.f / (1.f + expf(-x)) - y);
  }
  s_gate = a_gate;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s_mel += __shfl_xor_sync(0xffffffffu, s_mel, o);
    s_post += __shfl_xor_sync(0xffffffffu, s_post, o);
    s_gate += __shfl_xor_sync(0xffffffffu, s_gate, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = s_mel; red[1][w] = s_post; red[2][w] = s_gate; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double a = 0.0;
    for (int i = 0; i < 8; ++i) a += red[threadIdx.x][i];
    part[(long)threadIdx.x * gridDim.x + blockIdx.x] = a;
  }
}
__global__ void loss_final_kernel(const double* __restrict__ part, int nblk, double n_mel, double n_gate, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < nblk; ++i) s[k] += part[(long)k * nblk + i];
  out[1] = (float)(s[0] / n_mel); out[2] = (float)(s[1] / n_mel); out[3] = (float)(s[2] / n_gate);
  out[0] = out[1] + out[2] + out[3];     // summed in fp32 like the reference: (mel + post) + gate
}

double* loss_ws_layout(Carve& c) { return c.take<double>(3 * kLossSplit); }   // per-block partial sums

}  // namespace
}  // namespace t2

extern "C" {

size_t t2_loss_workspace_bytes(void) { t2::Carve c(nullptr); t2::loss_ws_layout(c); return c.bytes(); }

int t2_tacotron2_loss(const T2LossArgs* a, void* stream) {
  using namespace t2;
  if (!a || !a->mel || !a->mel_post || !a->gate || !a->mel_target || !a->gate_target || !a->loss || !a->ws)
    return fail(T2_ERR_INVALID, "loss: null argument");
  if (a->B <= 0 || a->C <= 0 || a->T <= 0) return fail(T2_ERR_INVALID, "loss: empty batch");
  if (a->ws_bytes < t2_loss_workspace_bytes()) return fail(T2_ERR_WORKSPACE, "loss workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  Carve c(a->ws);
  double* part = loss_ws_layout(c);
  const long n_mel = (long)a->B * a->C * a->T;
  int nblk = (int)((n_mel + 256 * 8 - 1) / (256 * 8));
  nblk = nblk < 1 ? 1 : (nblk > kLossSplit ? kLossSplit : nblk);
  loss_part_kernel<<<nblk, 256, 0, s>>>(a->mel, a->mel_post, a->gate, a->mel_target, a->gate_target, a->output_lengths, a->B, a->C,
                                        a->T, a->d_mel, a->d_mel_post, a->d_gate, part);
  T2_LAUNCH_CHECK();
  loss_final_kernel<<<1, 32, 0, s>>>(part, nblk, (double)n_mel, (double)a->B * a->T, a->loss);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
