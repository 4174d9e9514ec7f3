// fp32 SIMT GEMM (see gemm_f32.cuh).  64x64x16 tiles, 256 threads, 4x4 outputs per thread.
#include "gemm_f32.cuh"

namespace t2 {

__global__ void __launch_bounds__(256) gemm_f32_kernel(const GemmArgs a) {
  if (a.skip_flag != nullptr && *a.skip_flag != 0) return;
  __shared__ __align__(16) float As[16][64 + 4];
  __shared__ __align__(16) float Ws[16][64 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int am = m0 + lrow;
  const int wn = n0 + lrow;

  for (int s = 0; s < a.nseg; ++s) {
    const GemmSeg sg = a.seg[s];
    for (int k0 = 0; k0 < sg.K; k0 += 16) {
      float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
      if (am < a.M) av = *reinterpret_cast<const float4*>(sg.A + (long)am * sg.lda + k0 + lk);
      float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (wn < a.N) wv = *reinterpret_cast<const float4*>(sg.W + (long)wn * sg.ldw + k0 + lk);
      As[lk + 0][lrow] = av.x; As[lk + 1][lrow] = av.y; As[lk + 2][lrow] = av.z; As[lk + 3][lrow] = av.w;
      Ws[lk + 0][lrow] = wv.x; Ws[lk + 1][lrow] = wv.y; Ws[lk + 2][lrow] = wv.z; Ws[lk + 3][lrow] = wv.w;
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        const float4 af = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 wf = *reinterpret_cast<const float4*>(&Ws[kk][tx * 4]);
        const float ar[4] = {af.x, af.y, af.z, af.w};
        const float wr[4] = {wf.x, wf.y, wf.z, wf.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], wr[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  const float inv_keep = a.p_drop > 0.f ? 1.0f / (1.0f - a.p_drop) : 1.0f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= a.N) continue;
      float v = acc[i][j];
      if (a.bias) v += a.bias[n];
      if (a.act == ACT_RELU) v = fmaxf(v, 0.f);
      else if (a.act == ACT_TANH) v = tanhf(v);
      if (a.keep) v = a.keep[(long)m * a.ldkeep + n] ? v * inv_keep : 0.f;
      else if (a.philox) v = philox_keep(a.seed, a.site, (uint64_t)m * a.N + n, a.p_drop) ? v * inv_keep : 0.f;
      a.C[(long)m * a.ldc + n] = v;
    }
  }
}

int gemm_f32(const GemmArgs& a, cudaStream_t s) {
  if (a.M <= 0 || a.N <= 0) return T2_OK;
  for (int i = 0; i < a.nseg; ++i)
    if (a.seg[i].K % 16 != 0 || (a.seg[i].lda & 3) || (a.seg[i].ldw & 3))
      return fail(T2_ERR_INVALID, "gemm_f32: K %% 16 / ld %% 4 violated (seg %d: K=%d)", i, a.seg[i].K);
  dim3 grid((a.N + 63) / 64, (a.M + 63) / 64);
  gemm_f32_kernel<<<grid, 256, 0, s>>>(a);
  T2_LAUNCH_CHECK();
  return T2_OK;
}

}  // namespace t2
