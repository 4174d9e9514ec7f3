// Micro-benchmark of wgmma issue / execution cost on shared-memory-resident operands (no streaming):
// cycles for R back-to-back MMAs (m64nNk16, fp16 operands, fp32 accumulate) issued by one warpgroup, measured
// by its first thread from the first issue to the completion of the final commit group.  Drives the design notes
// in DESIGN.md.
#include "common.cuh"
#include "umma.cuh"

namespace t2 {
namespace {

// operands: A 128 rows x 64 k, B 256 rows x 64 k (SWIZZLE_128B images), contents irrelevant (finite)
__device__ __forceinline__ void fill_operands(uint8_t* smem) {
  for (int i = threadIdx.x; i < (128 + 256) * 64; i += 128) reinterpret_cast<__half*>(smem)[i] = __float2half(0.001f * (i & 63));
  ptx::fence_proxy_async();
  __syncthreads();
}

template <int N>
__device__ __forceinline__ void keep_alive(const float* d, long long* out) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s += d[i];
  if (s == 1234.5f) out[1] = -1;     // never true for these operands; keeps the MMAs from being optimised away
}

template <int N>
__global__ void __launch_bounds__(128, 1) mma_rate_kernel(int reps, int alternate_d, long long* out) {
  extern __shared__ __align__(1024) uint8_t smem[];
  fill_operands(smem);
  const uint32_t as = ptx::smem_u32(smem), bs = as + 128 * 128;
  float d0[N / 2], d1[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
  ptx::wg_fence_regs<N / 2>(d0);
  ptx::wg_fence_regs<N / 2>(d1);
  ptx::wg_fence();
  const long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    const int kk = r & 3;
    const uint64_t a = ptx::make_sw128_desc(as + kk * 32), b = ptx::make_sw128_desc(bs + kk * 32);
    if (alternate_d && (r & 1)) ptx::wgmma_f16<N>(d1, a, b);
    else ptx::wgmma_f16<N>(d0, a, b);
  }
  const long long t1 = clock64();
  ptx::wg_commit();
  ptx::wg_wait<0>();
  ptx::wg_fence_regs<N / 2>(d0);
  ptx::wg_fence_regs<N / 2>(d1);
  const long long t2 = clock64();
  if (threadIdx.x == 0) {
    out[0] = t1 - t0;   // issue time
    out[1] = t2 - t0;   // issue + drain
  }
  keep_alive<N>(d0, out);
  keep_alive<N>(d1, out);
}

// groups of `group` MMAs, each group followed by a commit + a wait for its completion (what one K chunk of a
// streaming event does): out[0] = cycles for `reps` groups, i.e. the cost of a COLD group incl. the wait round trip
template <int N>
__global__ void __launch_bounds__(128, 1) mma_group_kernel(int group, int reps, long long* out) {
  extern __shared__ __align__(1024) uint8_t smem[];
  fill_operands(smem);
  const uint32_t as = ptx::smem_u32(smem), bs = as + 128 * 128;
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  ptx::wg_fence_regs<N / 2>(d);
  const long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    ptx::wg_fence();
    for (int g = 0; g < group; ++g) {
      const int kk = g & 3;
      ptx::wgmma_f16<N>(d, ptx::make_sw128_desc(as + kk * 32), ptx::make_sw128_desc(bs + kk * 32));
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::wg_fence_regs<N / 2>(d);
  }
  if (threadIdx.x == 0) {
    out[0] = clock64() - t0;
    out[1] = 0;
  }
  keep_alive<N>(d, out);
}

constexpr size_t kBenchSmem = (128 + 256) * 128 + 1024;

int run_bench(void (*k)(int, int, long long*), int a0, int a1, long long* out_host, cudaStream_t s) {
  long long* d = nullptr;
  T2_CUDA(cudaMalloc((void**)&d, 16));
  T2_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBenchSmem));
  k<<<1, 128, kBenchSmem, s>>>(a0, a1, d);
  T2_LAUNCH_CHECK();
  T2_CUDA(cudaStreamSynchronize(s));
  T2_CUDA(cudaMemcpy(out_host, d, 16, cudaMemcpyDeviceToHost));
  cudaFree(d);
  return T2_OK;
}

}  // namespace

// M is the warpgroup's 64 rows; N in {32, 64, 128}
int mma_group(int M, int N, int group, int reps, long long* out_host, cudaStream_t s) {
  if (M != 64) return fail(T2_ERR_INVALID, "mma_group: M must be 64 (one warpgroup)");
  if (N == 32) return run_bench(mma_group_kernel<32>, group, reps, out_host, s);
  if (N == 64) return run_bench(mma_group_kernel<64>, group, reps, out_host, s);
  if (N == 128) return run_bench(mma_group_kernel<128>, group, reps, out_host, s);
  return fail(T2_ERR_INVALID, "mma_group: N in {32, 64, 128}");
}

int mma_rate(int M, int N, int reps, int alternate_d, long long* out_host, cudaStream_t s) {
  if (M != 64) return fail(T2_ERR_INVALID, "mma_rate: M must be 64 (one warpgroup)");
  if (N == 32) return run_bench(mma_rate_kernel<32>, reps, alternate_d, out_host, s);
  if (N == 64) return run_bench(mma_rate_kernel<64>, reps, alternate_d, out_host, s);
  if (N == 128) return run_bench(mma_rate_kernel<128>, reps, alternate_d, out_host, s);
  return fail(T2_ERR_INVALID, "mma_rate: N in {32, 64, 128}");
}

}  // namespace t2
