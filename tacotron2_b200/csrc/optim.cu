// Fused gradient clipping + Adam update (train.py:229-236: clip_grad_norm_ then torch.optim.Adam.step) as three
// multi-tensor launches over a chunk table: sum of squares -> global norm / clip coefficient -> in-place update of
// gradient (scaled, like clip_grad_norm_), exp_avg, exp_avg_sq and parameter.  fp32.
#include <cuda_fp16.h>
#include <math.h>

#include <vector>

#include "common.cuh"

namespace t2 {
namespace {

constexpr int kChunk = 32768;
struct Chunk { float* p; float* g; float* m; float* v; int n; };

__global__ void __launch_bounds__(256) sumsq_kernel(const Chunk* __restrict__ chunks, double* __restrict__ partial) {
  __shared__ float red[8];
  const Chunk c = chunks[blockIdx.x];
  float s = 0.f;
  for (int i = threadIdx.x; i < c.n; i += 256) { const float g = c.g[i]; s = fmaf(g, g, s); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < 8; ++i) a += (double)red[i];
    partial[blockIdx.x] = a;
  }
}
__global__ void norm_kernel(const double* __restrict__ partial, int n, float max_norm, float* __restrict__ out_norm, float* __restrict__ coef) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0;
  for (int i = 0; i < n; ++i) a += partial[i];
  const float norm = (float)sqrt(a);
  *out_norm = norm;
  float c = 1.f;
  if (max_norm > 0.f) { c = max_norm / (norm + 1e-6f); if (c > 1.f) c = 1.f; }   // torch.nn.utils.clip_grad_norm_
  *coef = c;
}
__global__ void __launch_bounds__(256) adam_kernel(const Chunk* __restrict__ chunks, const float* __restrict__ coef, float step_size, float beta1,
                                                   float beta2, float omb1, float omb2, float eps, float wd, float bc2_sqrt) {
  const Chunk c = chunks[blockIdx.x];
  const float k = *coef;
  for (int i = threadIdx.x; i < c.n; i += 256) {
    float g = c.g[i] * k;
    c.g[i] = g;                                   // clip_grad_norm_ scales .grad in place
    const float p = c.p[i];
    g = fmaf(wd, p, g);                           // Adam's L2 weight decay
    const float m = fmaf(beta1, c.m[i], omb1 * g);          // omb = 1 - beta, formed in double on the host
    const float v = fmaf(beta2, c.v[i], omb2 * g * g);
    c.m[i] = m; c.v[i] = v;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    c.p[i] = p - step_size * (m / denom);
  }
}


// ---- mixed precision (the reference's Apex AMP O2 flow, train.py:173-176, 222-236) ---------------------------------
// fp16 (or fp32) model parameters with fp32 masters, gradients multiplied by a dynamic loss scale, overflow => the step is
// skipped and the scale halved; growth_interval good steps => the scale doubles.  Everything -- unscale, overflow check,
// global-norm clip on the unscaled (master) gradients, Adam on the masters, fp16 write-back, scaler and step-count update --
// runs on the device in the same three multi-tensor launches: no host synchronisation, the host never learns whether a
// step was skipped unless it asks.
struct AmpChunk { void* p; const void* g; float* w; float* m; float* v; int n; int half_p; int half_g; };
// device-side optimizer state: [0] loss scale, [1] good steps since the last scale change, [2] optimizer steps taken
// (skipped steps do not count), [3] 1.0 if the last step was skipped
struct AmpDerived { float inv_scale, coef, step_size, bc2_sqrt; int skipped; };

__device__ __forceinline__ float amp_grad(const AmpChunk& c, int i) {
  return c.half_g ? __half2float(reinterpret_cast<const __half*>(c.g)[i]) : reinterpret_cast<const float*>(c.g)[i];
}
__global__ void __launch_bounds__(256) amp_sumsq_kernel(const AmpChunk* __restrict__ chunks, const float* __restrict__ state,
                                                        double* __restrict__ partial) {
  __shared__ float red[8];
  const AmpChunk c = chunks[blockIdx.x];
  const float inv = 1.f / state[0];
  float s = 0.f;
  for (int i = threadIdx.x; i < c.n; i += 256) { const float g = amp_grad(c, i) * inv; s = fmaf(g, g, s); }   // inf / nan propagate
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < 8; ++i) a += (double)red[i];
    partial[blockIdx.x] = a;
  }
}
__global__ void amp_norm_kernel(const double* __restrict__ partial, int n, float max_norm, double lr, double beta1, double beta2,
                                int growth_interval, float growth, float backoff, float* __restrict__ state,
                                float* __restrict__ out_norm, int* __restrict__ out_skipped, AmpDerived* __restrict__ d) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0;
  for (int i = 0; i < n; ++i) a += partial[i];
  const float norm = (float)sqrt(a);
  const bool bad = !isfinite(norm);
  *out_norm = norm;
  d->inv_scale = 1.f / state[0];                 // the scale the gradients of THIS step were multiplied with
  float c = 1.f;
  if (!bad && max_norm > 0.f) { c = max_norm / (norm + 1e-6f); if (c > 1.f) c = 1.f; }   // clip_grad_norm_ on the master gradients
  d->coef = c;
  d->skipped = bad ? 1 : 0;
  if (out_skipped) *out_skipped = d->skipped;
  if (bad) {                                     // apex.amp LossScaler.update_scale: overflow -> scale / 2, counter reset
    state[0] = fmaxf(state[0] * backoff, 1.f);
    state[1] = 0.f;
    state[3] = 1.f;
  } else {
    const double step = (double)state[2] + 1.0;  // torch.optim.Adam bias corrections for this step
    state[2] = (float)step;
    d->step_size = (float)(lr / (1.0 - pow(beta1, step)));
    d->bc2_sqrt = (float)sqrt(1.0 - pow(beta2, step));
    state[1] += 1.f;
    if (growth_interval > 0 && state[1] >= (float)growth_interval) { state[0] = fminf(state[0] * growth, 16777216.f); state[1] = 0.f; }
    state[3] = 0.f;
  }
}
__global__ void __launch_bounds__(256) amp_adam_kernel(const AmpChunk* __restrict__ chunks, const AmpDerived* __restrict__ d, float beta1,
                                                       float beta2, float omb1, float omb2, float eps, float wd) {
  if (d->skipped) return;                        // overflow: masters, moments and model weights stay as they are
  const AmpChunk c = chunks[blockIdx.x];
  const float k = d->inv_scale * d->coef, step_size = d->step_size, bc2_sqrt = d->bc2_sqrt;
  for (int i = threadIdx.x; i < c.n; i += 256) {
    float g = amp_grad(c, i) * k;
    const float w = c.w[i];
    g = fmaf(wd, w, g);
    const float m = fmaf(beta1, c.m[i], omb1 * g);
    const float v = fmaf(beta2, c.v[i], omb2 * g * g);
    c.m[i] = m; c.v[i] = v;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    const float nw = w - step_size * (m / denom);
    c.w[i] = nw;
    if (c.half_p) reinterpret_cast<__half*>(c.p)[i] = __float2half_rn(nw);     // master -> model copy (apex _master_params_to_model_params)
    else if (c.p != (void*)c.w) reinterpret_cast<float*>(c.p)[i] = nw;
  }
}

// per-chunk partial sums of squares, the derived scalars (Coef = float coefficient | AmpDerived), the chunk table
template <typename Coef, typename C>
void adam_ws_layout(Carve& c, size_t nchunk, double** partial, Coef** coef, C** chunks) {
  *partial = c.take<double>(nchunk);
  *coef = c.take<Coef>(1);
  *chunks = c.take<C>(nchunk);
}
// the chunk count is at most this bound, so the layout of the bound covers every call
inline size_t max_chunks(int64_t total_elements, int32_t n_tensors) {
  return (size_t)(total_elements / kChunk) + (size_t)n_tensors + 1;
}

}  // namespace
}  // namespace t2

extern "C" {

size_t t2_clip_adam_workspace_bytes(int64_t total_elements, int32_t n_tensors) {
  using namespace t2;
  Carve c(nullptr);
  double* partial; float* coef; Chunk* chunks;
  adam_ws_layout(c, max_chunks(total_elements, n_tensors), &partial, &coef, &chunks);
  return c.bytes();
}

int t2_clip_adam_step(const T2AdamArgs* a, void* stream) {
  using namespace t2;
  if (!a || a->n <= 0 || !a->params || !a->grads || !a->exp_avg || !a->exp_avg_sq || !a->numel || !a->grad_norm || !a->ws)
    return fail(T2_ERR_INVALID, "clip_adam: null argument");
  if (a->step < 1) return fail(T2_ERR_INVALID, "clip_adam: step counts from 1");
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<Chunk> chunks;
  int64_t total = 0;
  for (int t = 0; t < a->n; ++t) {
    total += a->numel[t];
    for (int64_t o = 0; o < a->numel[t]; o += kChunk) {
      Chunk c;
      c.p = a->params[t] + o; c.g = a->grads[t] + o; c.m = a->exp_avg[t] + o; c.v = a->exp_avg_sq[t] + o;
      c.n = (int)((a->numel[t] - o) < kChunk ? (a->numel[t] - o) : kChunk);
      chunks.push_back(c);
    }
  }
  if (a->ws_bytes < t2_clip_adam_workspace_bytes(total, a->n)) return fail(T2_ERR_WORKSPACE, "clip_adam workspace too small");
  const size_t nchunk = chunks.size();
  Carve c(a->ws);
  double* partial; float* coef; Chunk* d_chunks;
  adam_ws_layout(c, nchunk, &partial, &coef, &d_chunks);
  T2_CUDA(cudaMemcpyAsync(d_chunks, chunks.data(), nchunk * sizeof(Chunk), cudaMemcpyHostToDevice, s));   // pageable: staged before return
  sumsq_kernel<<<(unsigned)nchunk, 256, 0, s>>>(d_chunks, partial);
  T2_LAUNCH_CHECK();
  norm_kernel<<<1, 32, 0, s>>>(partial, (int)nchunk, (float)a->max_norm, a->grad_norm, coef);
  T2_LAUNCH_CHECK();
  const double bc1 = 1.0 - pow(a->beta1, (double)a->step), bc2 = 1.0 - pow(a->beta2, (double)a->step);
  adam_kernel<<<(unsigned)nchunk, 256, 0, s>>>(d_chunks, coef, (float)(a->lr / bc1), (float)a->beta1, (float)a->beta2, (float)(1.0 - a->beta1),
                                               (float)(1.0 - a->beta2), (float)a->eps,
                                               (float)a->weight_decay, (float)sqrt(bc2));
  T2_LAUNCH_CHECK();
  return T2_OK;
}

size_t t2_amp_adam_workspace_bytes(int64_t total_elements, int32_t n_tensors) {
  using namespace t2;
  Carve c(nullptr);
  double* partial; AmpDerived* derived; AmpChunk* chunks;
  adam_ws_layout(c, max_chunks(total_elements, n_tensors), &partial, &derived, &chunks);
  return c.bytes();
}

int t2_amp_adam_step(const T2AmpAdamArgs* a, void* stream) {
  using namespace t2;
  if (!a || a->n <= 0 || !a->model_params || !a->param_is_half || !a->grads || !a->grad_is_half || !a->master || !a->exp_avg ||
      !a->exp_avg_sq || !a->numel || !a->state || !a->grad_norm || !a->ws)
    return fail(T2_ERR_INVALID, "amp_adam: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<AmpChunk> chunks;
  int64_t total = 0;
  for (int t = 0; t < a->n; ++t) {
    total += a->numel[t];
    const int hp = a->param_is_half[t] ? 1 : 0, hg = a->grad_is_half[t] ? 1 : 0;
    for (int64_t o = 0; o < a->numel[t]; o += kChunk) {
      AmpChunk c;
      c.p = (char*)a->model_params[t] + o * (hp ? 2 : 4);
      c.g = (const char*)a->grads[t] + o * (hg ? 2 : 4);
      c.w = a->master[t] + o; c.m = a->exp_avg[t] + o; c.v = a->exp_avg_sq[t] + o;
      c.n = (int)((a->numel[t] - o) < kChunk ? (a->numel[t] - o) : kChunk);
      c.half_p = hp; c.half_g = hg;
      chunks.push_back(c);
    }
  }
  if (a->ws_bytes < t2_amp_adam_workspace_bytes(total, a->n)) return fail(T2_ERR_WORKSPACE, "amp_adam workspace too small");
  const size_t nchunk = chunks.size();
  Carve c(a->ws);
  double* partial; AmpDerived* derived; AmpChunk* d_chunks;
  adam_ws_layout(c, nchunk, &partial, &derived, &d_chunks);
  T2_CUDA(cudaMemcpyAsync(d_chunks, chunks.data(), nchunk * sizeof(AmpChunk), cudaMemcpyHostToDevice, s));
  amp_sumsq_kernel<<<(unsigned)nchunk, 256, 0, s>>>(d_chunks, a->state, partial);
  T2_LAUNCH_CHECK();
  amp_norm_kernel<<<1, 32, 0, s>>>(partial, (int)nchunk, (float)a->max_norm, a->lr, a->beta1, a->beta2, a->growth_interval,
                                   a->growth_factor, a->backoff_factor, a->state, a->grad_norm, a->skipped, derived);
  T2_LAUNCH_CHECK();
  amp_adam_kernel<<<(unsigned)nchunk, 256, 0, s>>>(d_chunks, derived, (float)a->beta1, (float)a->beta2, (float)(1.0 - a->beta1),
                                                   (float)(1.0 - a->beta2), (float)a->eps, (float)a->weight_decay);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // extern "C"
