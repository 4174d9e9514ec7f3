// Training path of the encoder / postnet (train_layers.cu): the conv stacks of every training-mode forward and every
// forward under autograd (with a stash, kept for the backward pass), and the backward.
// Without a stash the forward runs on `ws`, a region of postnet_forward_train_ws_bytes / encoder_convs_train_ws_bytes.
#pragma once
#include "model.h"

namespace t2 {

size_t postnet_stash_bytes(int B, int T);
size_t postnet_forward_train_ws_bytes(int B, int T);
int postnet_forward_train(T2Model* m, const T2PostnetArgs* a, void* ws, cudaStream_t s);
size_t postnet_backward_ws_bytes(int B, int T);
int postnet_backward(T2Model* m, const T2PostnetBwdArgs* a, cudaStream_t s);

size_t encoder_stash_bytes(int B, int T);
size_t encoder_convs_train_ws_bytes(int B, int T);
int encoder_convs_train(T2Model* m, const T2EncoderArgs* a, void* ws, cudaStream_t s, const float** xl, float** gates, float** cst);
int encoder_stash_output(const T2EncoderArgs* a, cudaStream_t s);
size_t encoder_backward_ws_bytes(int B, int T);
int encoder_backward(T2Model* m, const T2EncoderBwdArgs* a, cudaStream_t s);

}  // namespace t2
