// WaveGlow inference (waveglow.cu): host-side interface used by the C ABI in capi.cu.
#pragma once
#include "common.cuh"

struct T2WaveGlow;

namespace t2 {

int    waveglow_create(T2WaveGlow** out, const T2WaveGlowConfig* cfg, const void* const* weights, int n, cudaStream_t s);
int    waveglow_refresh(T2WaveGlow* h, const void* const* weights, int n, cudaStream_t s);
int    waveglow_destroy(T2WaveGlow* h);
size_t waveglow_ws_bytes(const T2WaveGlow* h, int B, int T_mel);
int    waveglow_infer(T2WaveGlow* h, const T2WaveGlowArgs* a, cudaStream_t s);
int    waveglow_infer_window(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, cudaStream_t s);
void   waveglow_window_halo(int* left, int* right);
int    waveglow_window_halo_config(const T2WaveGlowConfig* cfg, int* left, int* right);
int    waveglow_num_weights(const T2WaveGlowConfig* cfg);
#ifdef T2_SELFTEST
int    waveglow_state(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, int n_launches, float* spect, float* hbuf, float* acts,
                      float* skip, float* aud, cudaStream_t s);
#endif

}  // namespace t2
