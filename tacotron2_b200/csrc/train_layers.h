// Training path of the encoder / postnet (train_layers.cu): forward with stash + backward.
#pragma once
#include "model.h"

namespace t2 {

size_t postnet_stash_bytes(int B, int T);
int postnet_forward_train(T2Model* m, const T2PostnetArgs* a, cudaStream_t s);
size_t postnet_backward_ws_bytes(int B, int T);
int postnet_backward(T2Model* m, const T2PostnetBwdArgs* a, cudaStream_t s);

size_t encoder_stash_bytes(int B, int T);
int encoder_convs_train(T2Model* m, const T2EncoderArgs* a, cudaStream_t s, const float** xl, float** gates, float** cst);
int encoder_stash_output(const T2EncoderArgs* a, cudaStream_t s);
size_t encoder_backward_ws_bytes(int B, int T);
int encoder_backward(T2Model* m, const T2EncoderBwdArgs* a, cudaStream_t s);

}  // namespace t2
