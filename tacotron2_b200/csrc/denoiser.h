// WaveGlow denoiser, public STFT and Griffin-Lim (denoiser.cu): host-side interface used by the C ABI in capi.cu.
#pragma once
#include "common.cuh"

struct T2Denoiser;

namespace t2 {

int    denoiser_create(T2Denoiser** out, const T2DenoiserConfig* cfg, const float* forward_basis,
                       const float* inverse_basis, cudaStream_t s);
int    denoiser_refresh(T2Denoiser* h, const float* forward_basis, const float* inverse_basis, cudaStream_t s);
int    denoiser_destroy(T2Denoiser* h);
int    denoiser_bias(T2Denoiser* h, const float* audio, int n, float* bias_out, cudaStream_t s);
size_t denoiser_ws_bytes(int B, int n);
int    denoiser_run(T2Denoiser* h, const T2DenoiserArgs* a, cudaStream_t s);
int    denoiser_run_window(T2Denoiser* h, const T2DenoiserWindowArgs* a, cudaStream_t s);
void   denoiser_window_halo(int* left, int* right);
size_t stft_ws_bytes(int B, int n, bool signal);
int    stft_transform(T2Denoiser* h, const T2StftTransformArgs* a, cudaStream_t s);
int    stft_inverse(T2Denoiser* h, const T2StftInverseArgs* a, cudaStream_t s);
int    griffin_lim(T2Denoiser* h, const T2GriffinLimArgs* a, cudaStream_t s);

}  // namespace t2
