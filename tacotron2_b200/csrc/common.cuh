// Shared host/device helpers for libt2b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/t2b200.h"

namespace t2 {

// ---- error plumbing (thread-local message, negative return codes; nothing aborts) -------------
std::string& last_error();
int fail(int code, const char* fmt, ...);
extern long long g_launch_count;

#define T2_CUDA(expr)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return ::t2::fail(T2_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                               \
  } while (0)

#define T2_LAUNCH_CHECK()                                                                  \
  do {                                                                                     \
    ::t2::g_launch_count++;                                                                \
    cudaError_t _e = cudaGetLastError();                                                   \
    if (_e != cudaSuccess)                                                                 \
      return ::t2::fail(T2_ERR_CUDA, "kernel launch failed: %s (%s:%d)",                   \
                        cudaGetErrorString(_e), __FILE__, __LINE__);                       \
  } while (0)

#define T2_TRY(expr)             \
  do {                           \
    int _r = (expr);             \
    if (_r != T2_OK) return _r;  \
  } while (0)

// ---- model dimensions the kernels are specialised for (hparams.py:40-75 defaults) -------------
constexpr int kMel = 80;
constexpr int kEnc = 512;       // encoder_embedding_dim (memory width)
constexpr int kARnn = 1024;     // attention_rnn_dim
constexpr int kDRnn = 1024;     // decoder_rnn_dim
constexpr int kPre = 256;       // prenet_dim
constexpr int kAtt = 128;       // attention_dim
constexpr int kLocF = 32;       // attention_location_n_filters
constexpr int kLocK = 31;       // attention_location_kernel_size
constexpr int kPost = 512;      // postnet_embedding_dim
constexpr int kConvK = 5;       // encoder / postnet kernel size
constexpr int kEncH = 256;      // encoder LSTM hidden per direction

// state_dict order (tests/common.state_dict_shapes; SURVEY.md section 8(b1))
enum W : int {
  W_EMB = 0,
  // encoder.convolutions.{i}: conv.weight, conv.bias, bn.weight, bn.bias, running_mean,
  // running_var, num_batches_tracked  (7 entries each, i = 0..2)
  W_ENC_CONV0 = 1,
  W_ENC_LSTM = 22,  // weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0, then *_reverse (8)
  W_PRENET0 = 30,
  W_PRENET1 = 31,
  W_ARNN_WIH = 32, W_ARNN_WHH = 33, W_ARNN_BIH = 34, W_ARNN_BHH = 35,
  W_ATT_QUERY = 36, W_ATT_MEMORY = 37, W_ATT_V = 38, W_ATT_LOC_CONV = 39, W_ATT_LOC_DENSE = 40,
  W_DRNN_WIH = 41, W_DRNN_WHH = 42, W_DRNN_BIH = 43, W_DRNN_BHH = 44,
  W_PROJ_W = 45, W_PROJ_B = 46, W_GATE_W = 47, W_GATE_B = 48,
  W_POST_CONV0 = 49,  // 5 x 7 entries
  W_COUNT = 84
};
static_assert(W_POST_CONV0 + 5 * 7 == W_COUNT, "state_dict table");

// ---- buffer layouts ------------------------------------------------------------------------------
// Bump allocator over one buffer.  Each buffer has one layout function that take()s its regions in order; the size
// query runs it on a null base, where it only measures (take() then returns the region's offset), and the code that
// uses the buffer runs it on the real base, so the two cannot disagree.  The base is first aligned up to `max_align`, the largest alignment
// the layout asks for, so both runs produce the same offsets whatever the caller's alignment; bytes() includes that
// reserve.  Alignments are powers of two.
struct Carve {
  char* base;
  size_t off = 0, max_align;
  __host__ __device__ __forceinline__ explicit Carve(void* b, size_t max_align = 256)
      : base((char*)b + (-(uintptr_t)b & (max_align - 1))), max_align(max_align) {}
  template <typename T>
  __host__ __device__ __forceinline__ T* take(size_t count, size_t align = 256) {
    off = (off + align - 1) & ~(align - 1);
    T* r = reinterpret_cast<T*>(base + off);
    off += count * sizeof(T);
    return r;
  }
  __host__ __device__ __forceinline__ size_t bytes() const { return off + max_align - 1; }
};

// ---- Philox4x32-10 (counter based RNG for the production dropout path) -------------------------
__host__ __device__ inline void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
    uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
    uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Bernoulli keep decision for element `idx` of dropout site `site` (a per-call unique id) with
// drop probability p: one Philox block serves 4 consecutive elements.
__host__ __device__ inline bool philox_keep(uint64_t seed, uint32_t site, uint64_t idx, float p) {
  uint32_t o[4];
  uint64_t blk = idx >> 2;
  philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), site, 0x7ac07201u, (uint32_t)seed,
                (uint32_t)(seed >> 32), o);
  float u = (float)(o[idx & 3] >> 8) * (1.0f / 16777216.0f);
  return u >= p;
}

}  // namespace t2
