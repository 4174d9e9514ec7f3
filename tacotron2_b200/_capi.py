"""ctypes binding of libt2b200.so (include/t2b200.h).  Importing this module never touches CUDA;
``lib()`` loads the shared library and raises loudly when it is missing -- there is NO CPU or
PyTorch fallback for the hot path.  ``call`` runs a library entry point on torch's current stream, and ``Workspace``
caches the device buffers the entry points take."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("T2B200_LIB") or os.path.join(_HERE, "libt2b200.so")   # T2B200_LIB: A/B test builds

T2_NUM_WEIGHTS = 84
IMPL_AUTO, IMPL_STEPWISE, IMPL_PERSISTENT = 0, 1, 2
MODE_INFER, MODE_TEACHER = 0, 1
DURATIONS_MAS, DURATIONS_ARGMAX = 0, 1
DURATIONS_MAX_TEXT = 4096           # T2_DURATIONS_MAX_TEXT
PYIN_MAX_FRAME, PYIN_MAX_BINS, PYIN_MAX_THRESHOLDS = 2048, 1536, 4096   # T2_PYIN_MAX_*
DTW_MAX_FRAMES, DTW_MAX_DIM = 8192, 1024                                # T2_DTW_MAX_FRAMES, T2_DTW_MAX_DIM
DTW_F32, DTW_F64 = 0, 1

EXPORTS = [
    "t2_abi_version", "t2_last_error", "t2_device_info", "t2_model_create", "t2_model_refresh",
    "t2_model_destroy", "t2_encoder_workspace_bytes", "t2_encoder_forward",
    "t2_decoder_workspace_bytes", "t2_decoder_run", "t2_prenet_forward",
    "t2_postnet_workspace_bytes", "t2_postnet_forward", "t2_infer_workspace_bytes", "t2_infer_host",
    "t2_encoder_infer", "t2_postnet_infer",
    "t2_kernel_launch_count", "t2_decoder_profile",
    "t2_decoder_stash_bytes", "t2_decoder_backward_workspace_bytes", "t2_decoder_backward",
    "t2_prenet_backward_workspace_bytes", "t2_prenet_backward",
    "t2_encoder_stash_bytes", "t2_encoder_backward_workspace_bytes", "t2_encoder_backward",
    "t2_postnet_stash_bytes", "t2_postnet_backward_workspace_bytes", "t2_postnet_backward",
    "t2_clip_adam_workspace_bytes", "t2_clip_adam_step", "t2_amp_adam_workspace_bytes", "t2_amp_adam_step",
    "t2_loss_workspace_bytes", "t2_tacotron2_loss",
    "t2_mel_spectrogram_frames", "t2_mel_spectrogram_workspace_bytes", "t2_mel_spectrogram", "t2_collate",
    "t2_mel_spectrogram_workspace_bytes_lengths",
    "t2_decoder_stream_state_bytes", "t2_decoder_stream_begin", "t2_decoder_stream_run",
    "t2_decoder_stream_admit", "t2_decoder_stream_collect",
    "t2_waveglow_create", "t2_waveglow_refresh", "t2_waveglow_destroy", "t2_waveglow_workspace_bytes",
    "t2_waveglow_infer", "t2_waveglow_infer_window", "t2_waveglow_window_halo", "t2_waveglow_window_halo_config",
    "t2_waveglow_num_weights",
    "t2_denoiser_create", "t2_denoiser_refresh", "t2_denoiser_destroy", "t2_denoiser_bias",
    "t2_denoiser_workspace_bytes", "t2_denoiser_run", "t2_denoiser_run_window", "t2_denoiser_window_halo",
    "t2_stft_transform_workspace_bytes", "t2_stft_transform", "t2_stft_inverse_workspace_bytes", "t2_stft_inverse",
    "t2_griffin_lim_workspace_bytes", "t2_griffin_lim",
    "t2_durations_workspace_bytes", "t2_durations",
    "t2_pyin_workspace_bytes", "t2_pyin", "t2_average_by_durations",
    "t2_dtw_workspace_bytes", "t2_dtw", "t2_mel_cepstra",
    "t2_decoder_step_workspace_bytes", "t2_decoder_step", "t2_attention_forward", "t2_processed_memory",
    "t2_hifigan_num_weights", "t2_hifigan_create", "t2_hifigan_refresh", "t2_hifigan_destroy",
    "t2_hifigan_workspace_bytes", "t2_hifigan_infer",
]
T2_WAVEGLOW_NUM_WEIGHTS = 686       # the published configuration's; t2_waveglow_num_weights gives any other's


class T2Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mel_channels", "n_symbols", "symbols_embedding_dim", "encoder_kernel_size",
        "encoder_n_convolutions", "encoder_embedding_dim", "attention_rnn_dim", "decoder_rnn_dim",
        "prenet_dim", "attention_dim", "attention_location_n_filters",
        "attention_location_kernel_size", "postnet_embedding_dim", "postnet_kernel_size",
        "postnet_n_convolutions")] + [("p_attention_dropout", C.c_float),
                                      ("p_decoder_dropout", C.c_float), ("bn_eps", C.c_float)]


class T2EncoderArgs(C.Structure):
    _fields_ = [("text", C.c_void_p), ("embedded", C.c_void_p), ("lengths", C.c_void_p), ("B", C.c_int32), ("T", C.c_int32),
                ("training", C.c_int32), ("keep", C.c_void_p), ("seed", C.c_uint64),
                ("memory", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t),
                ("stash", C.c_void_p), ("stash_bytes", C.c_size_t)]


class T2EncoderBwdArgs(C.Structure):
    _fields_ = [("text", C.c_void_p), ("embedded", C.c_void_p), ("lengths", C.c_void_p), ("B", C.c_int32), ("T", C.c_int32),
                ("training", C.c_int32), ("keep", C.c_void_p), ("seed", C.c_uint64),
                ("stash", C.c_void_p), ("stash_bytes", C.c_size_t), ("d_memory", C.c_void_p), ("d_embedded", C.c_void_p),
                ("grads", C.POINTER(C.c_void_p)), ("n_grads", C.c_int32), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2InferArgs(C.Structure):
    _fields_ = [("text_host", C.c_void_p), ("input_lengths_host", C.c_void_p), ("B", C.c_int32), ("T_text", C.c_int32),
                ("max_steps", C.c_int32), ("gate_threshold", C.c_float), ("seed", C.c_uint64), ("impl", C.c_int32),
                ("mel_post_host", C.c_void_p), ("mel_lengths_host", C.c_void_p), ("n_steps_host", C.c_void_p),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t), ("row_seeds_host", C.c_void_p)]


class T2DecoderArgs(C.Structure):
    _fields_ = [("mode", C.c_int32), ("impl", C.c_int32), ("training", C.c_int32),
                ("memory", C.c_void_p), ("memory_lengths", C.c_void_p),
                ("B", C.c_int32), ("T_enc", C.c_int32), ("n_steps_cap", C.c_int32),
                ("teacher_prenet", C.c_void_p), ("prenet_keep", C.c_void_p),
                ("att_keep", C.c_void_p), ("dec_keep", C.c_void_p), ("seed", C.c_uint64),
                ("gate_threshold", C.c_float), ("score_mask_value", C.c_float),
                ("mel", C.c_void_p), ("gate", C.c_void_p), ("align", C.c_void_p),
                ("mel_lengths", C.c_void_p), ("n_steps", C.c_void_p),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t),
                ("stash", C.c_void_p), ("stash_bytes", C.c_size_t), ("row_seeds", C.c_void_p),
                ("forced_align", C.c_void_p), ("forced_lengths", C.c_void_p),
                ("window_back", C.c_int32), ("window_front", C.c_int32), ("max_steps", C.c_void_p)]


class T2DecoderStepArgs(C.Structure):
    _fields_ = [("B", C.c_int32), ("T_enc", C.c_int32),
                ("memory", C.c_void_p), ("processed_memory", C.c_void_p), ("mask", C.c_void_p),
                ("attention_hidden", C.c_void_p), ("attention_cell", C.c_void_p), ("decoder_hidden", C.c_void_p),
                ("decoder_cell", C.c_void_p), ("attention_weights", C.c_void_p), ("attention_weights_cum", C.c_void_p),
                ("attention_context", C.c_void_p), ("decoder_input", C.c_void_p), ("mel", C.c_void_p), ("gate", C.c_void_p),
                ("training", C.c_int32), ("att_keep", C.c_void_p), ("dec_keep", C.c_void_p), ("seed", C.c_uint64),
                ("score_mask_value", C.c_float), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2AttentionArgs(C.Structure):
    _fields_ = [("B", C.c_int32), ("T_enc", C.c_int32), ("query", C.c_void_p), ("memory", C.c_void_p),
                ("processed_memory", C.c_void_p), ("attention_weights_cat", C.c_void_p), ("mask", C.c_void_p),
                ("score_mask_value", C.c_float), ("energies", C.c_void_p), ("location", C.c_void_p),
                ("weights", C.c_void_p), ("context", C.c_void_p)]


class T2DecoderStreamArgs(C.Structure):
    _fields_ = [("dec", T2DecoderArgs), ("state", C.c_void_p), ("state_bytes", C.c_size_t), ("status", C.c_void_p),
                ("row_step0", C.c_void_p)]


class T2CollectRow(C.Structure):
    _fields_ = [("row", C.c_int32), ("n_frames", C.c_int32), ("T_text", C.c_int32), ("reserved", C.c_int32),
                ("mel", C.c_void_p), ("gate", C.c_void_p), ("align", C.c_void_p)]


class T2DecoderBwdArgs(C.Structure):
    _fields_ = [("memory", C.c_void_p), ("memory_lengths", C.c_void_p),
                ("B", C.c_int32), ("T_enc", C.c_int32), ("T_mel", C.c_int32), ("training", C.c_int32),
                ("teacher_prenet", C.c_void_p), ("att_keep", C.c_void_p), ("dec_keep", C.c_void_p),
                ("seed", C.c_uint64), ("score_mask_value", C.c_float), ("align", C.c_void_p),
                ("stash", C.c_void_p), ("stash_bytes", C.c_size_t),
                ("d_mel", C.c_void_p), ("d_gate", C.c_void_p), ("d_align", C.c_void_p),
                ("d_memory", C.c_void_p), ("d_prenet", C.c_void_p),
                ("grads", C.POINTER(C.c_void_p)), ("n_grads", C.c_int32),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2PrenetBwdArgs(C.Structure):
    _fields_ = [("frames", C.c_void_p), ("M", C.c_int32), ("keep", C.c_void_p), ("seed", C.c_uint64),
                ("d_out", C.c_void_p), ("grads", C.POINTER(C.c_void_p)), ("n_grads", C.c_int32),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2AdamArgs(C.Structure):
    _fields_ = [("n", C.c_int32), ("params", C.POINTER(C.c_void_p)), ("grads", C.POINTER(C.c_void_p)),
                ("exp_avg", C.POINTER(C.c_void_p)), ("exp_avg_sq", C.POINTER(C.c_void_p)), ("numel", C.POINTER(C.c_int64)),
                ("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("max_norm", C.c_double), ("step", C.c_int32),
                ("grad_norm", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2AmpAdamArgs(C.Structure):
    _fields_ = [("n", C.c_int32), ("model_params", C.POINTER(C.c_void_p)), ("param_is_half", C.POINTER(C.c_int32)),
                ("grads", C.POINTER(C.c_void_p)), ("grad_is_half", C.POINTER(C.c_int32)),
                ("master", C.POINTER(C.c_void_p)), ("exp_avg", C.POINTER(C.c_void_p)), ("exp_avg_sq", C.POINTER(C.c_void_p)),
                ("numel", C.POINTER(C.c_int64)),
                ("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("max_norm", C.c_double),
                ("growth_interval", C.c_int32), ("growth_factor", C.c_float), ("backoff_factor", C.c_float),
                ("state", C.c_void_p), ("grad_norm", C.c_void_p), ("skipped", C.c_void_p),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2LossArgs(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("mel_post", C.c_void_p), ("gate", C.c_void_p), ("mel_target", C.c_void_p),
                ("gate_target", C.c_void_p), ("output_lengths", C.c_void_p), ("B", C.c_int32), ("C", C.c_int32), ("T", C.c_int32),
                ("loss", C.c_void_p), ("d_mel", C.c_void_p), ("d_mel_post", C.c_void_p), ("d_gate", C.c_void_p),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2MelSpecArgs(C.Structure):
    _fields_ = [("y", C.c_void_p), ("B", C.c_int32), ("n_samples", C.c_int32), ("filter_length", C.c_int32),
                ("hop_length", C.c_int32), ("n_mel", C.c_int32), ("forward_basis", C.c_void_p), ("mel_basis", C.c_void_p),
                ("clip_val", C.c_float), ("mel", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t),
                ("lengths", C.c_void_p)]


class T2CollateArgs(C.Structure):
    _fields_ = [("text_flat", C.c_void_p), ("text_offsets", C.c_void_p), ("mel_flat", C.c_void_p), ("mel_offsets", C.c_void_p),
                ("B", C.c_int32), ("n_mel", C.c_int32), ("T_max", C.c_int32), ("L_pad", C.c_int32), ("order", C.c_void_p),
                ("text_padded", C.c_void_p), ("input_lengths", C.c_void_p), ("mel_padded", C.c_void_p),
                ("gate_padded", C.c_void_p), ("output_lengths", C.c_void_p)]


class T2DurationsArgs(C.Structure):
    _fields_ = [("alignments", C.c_void_p), ("input_lengths", C.c_void_p), ("mel_lengths", C.c_void_p),
                ("B", C.c_int32), ("T_mel", C.c_int32), ("T_text", C.c_int32), ("method", C.c_int32),
                ("durations", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2PyinArgs(C.Structure):
    _fields_ = [("y", C.c_void_p), ("lengths", C.c_void_p)] + [
        (n, C.c_int32) for n in ("B", "n", "sr", "frame_length", "win_length", "hop_length", "min_period",
                                 "max_period", "n_thresholds", "n_bins", "bins_per_semitone", "width")] + [
        (n, C.c_double) for n in ("fmin", "no_trough_prob", "fill_na", "log_tiny", "log_init_unvoiced")] + [
        (n, C.c_void_p) for n in ("thresholds", "beta_probs", "beta_prefix", "boltzmann", "log_trans", "freqs",
                                  "f0", "voiced_flag", "voiced_prob", "ws")] + [("ws_bytes", C.c_size_t)]


class T2DtwArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("x_lengths", C.c_void_p), ("y_lengths", C.c_void_p)] + [
        (n, C.c_int32) for n in ("B", "D", "T_x", "T_y", "dtype")] + [
        (n, C.c_void_p) for n in ("cost", "path", "path_lengths", "ws")] + [("ws_bytes", C.c_size_t)]


class T2PostnetArgs(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("mel_batch_stride", C.c_int64), ("lengths", C.c_void_p),
                ("B", C.c_int32), ("T", C.c_int32), ("training", C.c_int32), ("keep", C.c_void_p),
                ("seed", C.c_uint64), ("add_residual", C.c_int32), ("mel_post", C.c_void_p), ("ws", C.c_void_p),
                ("ws_bytes", C.c_size_t), ("stash", C.c_void_p), ("stash_bytes", C.c_size_t)]


class T2PostnetBwdArgs(C.Structure):
    _fields_ = [("B", C.c_int32), ("T", C.c_int32), ("training", C.c_int32), ("add_residual", C.c_int32),
                ("keep", C.c_void_p), ("seed", C.c_uint64), ("wgrad_lengths", C.c_void_p),
                ("stash", C.c_void_p), ("stash_bytes", C.c_size_t),
                ("d_mel_post", C.c_void_p), ("d_mel", C.c_void_p),
                ("grads", C.POINTER(C.c_void_p)), ("n_grads", C.c_int32), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2WaveGlowConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mel_channels", "n_flows", "n_group", "n_early_every", "n_early_size", "wn_n_layers", "wn_kernel_size",
        "wn_n_channels", "fp16")]


class T2WaveGlowArgs(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("B", C.c_int32), ("T_mel", C.c_int32), ("lengths", C.c_void_p),
                ("io_half", C.c_int32), ("sigma", C.c_float), ("z", C.c_void_p), ("seed", C.c_uint64),
                ("audio", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t), ("row_seeds", C.c_void_p)]


class T2WaveGlowWindowArgs(C.Structure):
    _fields_ = [("wg", T2WaveGlowArgs), ("frame0", C.c_int32), ("out0", C.c_int32), ("out1", C.c_int32),
                ("z_frames", C.c_int32), ("at_end", C.c_int32)]


class T2HiFiGANConfig(C.Structure):
    _fields_ = [("n_mel_channels", C.c_int32), ("resblock", C.c_int32), ("n_upsamples", C.c_int32),
                ("upsample_rates", C.c_int32 * 8), ("upsample_kernel_sizes", C.c_int32 * 8),
                ("upsample_initial_channel", C.c_int32), ("n_kernels", C.c_int32),
                ("resblock_kernel_sizes", C.c_int32 * 8), ("resblock_dilation_sizes", (C.c_int32 * 3) * 8),
                ("fp16", C.c_int32)]


class T2HiFiGANArgs(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("B", C.c_int32), ("T_mel", C.c_int32), ("lengths", C.c_void_p),
                ("io_half", C.c_int32), ("audio", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2DenoiserConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("filter_length", "hop_length", "win_length", "window")]


class T2DenoiserArgs(C.Structure):
    _fields_ = [("audio", C.c_void_p), ("B", C.c_int32), ("n", C.c_int32), ("lengths", C.c_void_p),
                ("io_half", C.c_int32), ("bias", C.c_void_p), ("strength", C.c_float), ("out", C.c_void_p),
                ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2DenoiserWindowArgs(C.Structure):
    _fields_ = [("dn", T2DenoiserArgs), ("s0", C.c_int32), ("out0", C.c_int32), ("out1", C.c_int32),
                ("at_end", C.c_int32)]


class T2StftTransformArgs(C.Structure):
    _fields_ = [("audio", C.c_void_p), ("B", C.c_int32), ("n", C.c_int32), ("lengths", C.c_void_p),
                ("magnitude", C.c_void_p), ("phase", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2StftInverseArgs(C.Structure):
    _fields_ = [("magnitude", C.c_void_p), ("phase", C.c_void_p), ("B", C.c_int32), ("F", C.c_int32),
                ("lengths", C.c_void_p), ("out", C.c_void_p), ("ws", C.c_void_p), ("ws_bytes", C.c_size_t)]


class T2GriffinLimArgs(C.Structure):
    _fields_ = [("inv", T2StftInverseArgs), ("n_iters", C.c_int32)]


_lib = None


def lib():
    """The loaded shared library (raises RuntimeError if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(
            "tacotron2_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C tacotron2_b200/csrc`).  There is no CPU / PyTorch fallback "
            "for the hot path." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.t2_abi_version.restype = C.c_int
    L.t2_last_error.restype = C.c_char_p
    L.t2_kernel_launch_count.restype = C.c_int64
    L.t2_device_info.argtypes = [C.POINTER(C.c_int32)]
    L.t2_model_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(T2Config), C.POINTER(C.c_void_p),
                                  C.c_int32, C.c_void_p]
    L.t2_model_refresh.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p]
    L.t2_model_destroy.argtypes = [C.c_void_p]
    for n in ("t2_encoder_workspace_bytes", "t2_postnet_workspace_bytes", "t2_encoder_stash_bytes",
              "t2_encoder_backward_workspace_bytes", "t2_postnet_stash_bytes", "t2_postnet_backward_workspace_bytes"):
        getattr(L, n).restype = C.c_size_t
        getattr(L, n).argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    for n in ("t2_decoder_workspace_bytes", "t2_infer_workspace_bytes", "t2_decoder_stash_bytes",
              "t2_decoder_backward_workspace_bytes"):
        getattr(L, n).restype = C.c_size_t
        getattr(L, n).argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    L.t2_encoder_forward.argtypes = [C.c_void_p, C.POINTER(T2EncoderArgs), C.c_void_p]
    L.t2_encoder_infer.argtypes = [C.c_void_p, C.POINTER(T2EncoderArgs), C.c_void_p]
    L.t2_decoder_run.argtypes = [C.c_void_p, C.POINTER(T2DecoderArgs), C.c_void_p]
    L.t2_decoder_step_workspace_bytes.restype = C.c_size_t
    L.t2_decoder_step_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    L.t2_decoder_step.argtypes = [C.c_void_p, C.POINTER(T2DecoderStepArgs), C.c_void_p]
    L.t2_attention_forward.argtypes = [C.c_void_p, C.POINTER(T2AttentionArgs), C.c_void_p]
    L.t2_processed_memory.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    L.t2_decoder_stream_state_bytes.restype = C.c_size_t
    L.t2_decoder_stream_state_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.t2_decoder_stream_begin.argtypes = [C.c_void_p, C.POINTER(T2DecoderStreamArgs), C.c_void_p]
    L.t2_decoder_stream_run.argtypes = [C.c_void_p, C.POINTER(T2DecoderStreamArgs), C.c_int32, C.c_void_p, C.c_void_p]
    L.t2_decoder_stream_admit.argtypes = [C.c_void_p, C.POINTER(T2DecoderStreamArgs), C.POINTER(C.c_int32), C.c_int32,
                                          C.c_void_p]
    L.t2_decoder_stream_collect.argtypes = [C.c_void_p, C.POINTER(T2DecoderStreamArgs), C.POINTER(T2CollectRow), C.c_int32,
                                            C.c_void_p]
    L.t2_postnet_forward.argtypes = [C.c_void_p, C.POINTER(T2PostnetArgs), C.c_void_p]
    L.t2_postnet_infer.argtypes = [C.c_void_p, C.POINTER(T2PostnetArgs), C.c_void_p]
    L.t2_clip_adam_workspace_bytes.restype = C.c_size_t
    L.t2_clip_adam_workspace_bytes.argtypes = [C.c_int64, C.c_int32]
    L.t2_clip_adam_step.argtypes = [C.POINTER(T2AdamArgs), C.c_void_p]
    L.t2_amp_adam_workspace_bytes.restype = C.c_size_t
    L.t2_amp_adam_workspace_bytes.argtypes = [C.c_int64, C.c_int32]
    L.t2_amp_adam_step.argtypes = [C.POINTER(T2AmpAdamArgs), C.c_void_p]
    L.t2_loss_workspace_bytes.restype = C.c_size_t
    L.t2_loss_workspace_bytes.argtypes = []
    L.t2_tacotron2_loss.argtypes = [C.POINTER(T2LossArgs), C.c_void_p]
    L.t2_mel_spectrogram_frames.argtypes = [C.c_int32, C.c_int32]
    L.t2_mel_spectrogram_workspace_bytes.restype = C.c_size_t
    L.t2_mel_spectrogram_workspace_bytes.argtypes = [C.c_int32] * 5
    L.t2_mel_spectrogram_workspace_bytes_lengths.restype = C.c_size_t
    L.t2_mel_spectrogram_workspace_bytes_lengths.argtypes = [C.c_int32] * 5
    L.t2_mel_spectrogram.argtypes = [C.POINTER(T2MelSpecArgs), C.c_void_p]
    L.t2_collate.argtypes = [C.POINTER(T2CollateArgs), C.c_void_p]
    L.t2_encoder_backward.argtypes = [C.c_void_p, C.POINTER(T2EncoderBwdArgs), C.c_void_p]
    L.t2_postnet_backward.argtypes = [C.c_void_p, C.POINTER(T2PostnetBwdArgs), C.c_void_p]
    L.t2_decoder_backward.argtypes = [C.c_void_p, C.POINTER(T2DecoderBwdArgs), C.c_void_p]
    L.t2_prenet_backward.argtypes = [C.c_void_p, C.POINTER(T2PrenetBwdArgs), C.c_void_p]
    L.t2_prenet_backward_workspace_bytes.restype = C.c_size_t
    L.t2_prenet_backward_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    L.t2_prenet_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64,
                                    C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.t2_infer_host.argtypes = [C.c_void_p, C.POINTER(T2InferArgs), C.c_void_p]
    L.t2_decoder_profile.argtypes = [C.POINTER(T2DecoderArgs), C.POINTER(C.c_int64)]
    L.t2_waveglow_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(T2WaveGlowConfig), C.POINTER(C.c_void_p),
                                     C.c_int32, C.c_void_p]
    L.t2_waveglow_refresh.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p]
    L.t2_waveglow_destroy.argtypes = [C.c_void_p]
    L.t2_waveglow_workspace_bytes.restype = C.c_size_t
    L.t2_waveglow_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.t2_waveglow_infer.argtypes = [C.c_void_p, C.POINTER(T2WaveGlowArgs), C.c_void_p]
    L.t2_waveglow_infer_window.argtypes = [C.c_void_p, C.POINTER(T2WaveGlowWindowArgs), C.c_void_p]
    L.t2_waveglow_window_halo.restype = None
    L.t2_waveglow_window_halo.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.t2_waveglow_window_halo_config.argtypes = [C.POINTER(T2WaveGlowConfig), C.POINTER(C.c_int32),
                                                 C.POINTER(C.c_int32)]
    L.t2_waveglow_num_weights.restype = C.c_int32
    L.t2_waveglow_num_weights.argtypes = [C.POINTER(T2WaveGlowConfig)]
    L.t2_denoiser_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(T2DenoiserConfig), C.c_void_p, C.c_void_p,
                                     C.c_void_p]
    L.t2_denoiser_refresh.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.t2_denoiser_destroy.argtypes = [C.c_void_p]
    L.t2_denoiser_bias.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.t2_denoiser_workspace_bytes.restype = C.c_size_t
    L.t2_denoiser_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.t2_denoiser_run.argtypes = [C.c_void_p, C.POINTER(T2DenoiserArgs), C.c_void_p]
    L.t2_denoiser_run_window.argtypes = [C.c_void_p, C.POINTER(T2DenoiserWindowArgs), C.c_void_p]
    L.t2_denoiser_window_halo.restype = None
    L.t2_denoiser_window_halo.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    for n, args in (("t2_stft_transform", T2StftTransformArgs), ("t2_stft_inverse", T2StftInverseArgs),
                    ("t2_griffin_lim", T2GriffinLimArgs)):
        getattr(L, n + "_workspace_bytes").restype = C.c_size_t
        getattr(L, n + "_workspace_bytes").argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        getattr(L, n).argtypes = [C.c_void_p, C.POINTER(args), C.c_void_p]
    L.t2_durations_workspace_bytes.restype = C.c_size_t
    L.t2_durations_workspace_bytes.argtypes = [C.c_int32] * 4
    L.t2_durations.argtypes = [C.POINTER(T2DurationsArgs), C.c_void_p]
    L.t2_pyin_workspace_bytes.restype = C.c_size_t
    L.t2_pyin_workspace_bytes.argtypes = [C.POINTER(T2PyinArgs)]
    L.t2_pyin.argtypes = [C.POINTER(T2PyinArgs), C.c_void_p]
    L.t2_average_by_durations.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_void_p]
    L.t2_dtw_workspace_bytes.restype = C.c_size_t
    L.t2_dtw_workspace_bytes.argtypes = [C.c_int32] * 5
    L.t2_dtw.argtypes = [C.POINTER(T2DtwArgs), C.c_void_p]
    L.t2_mel_cepstra.argtypes = [C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p, C.c_int32,
                                                                                         C.c_void_p, C.c_void_p]
    L.t2_hifigan_num_weights.restype = C.c_int32
    L.t2_hifigan_num_weights.argtypes = [C.POINTER(T2HiFiGANConfig)]
    L.t2_hifigan_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(T2HiFiGANConfig), C.POINTER(C.c_void_p),
                                    C.c_int32, C.c_void_p]
    L.t2_hifigan_refresh.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p]
    L.t2_hifigan_destroy.argtypes = [C.c_void_p]
    L.t2_hifigan_workspace_bytes.restype = C.c_size_t
    L.t2_hifigan_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.t2_hifigan_infer.argtypes = [C.c_void_p, C.POINTER(T2HiFiGANArgs), C.c_void_p]
    if L.t2_abi_version() != 2:
        raise RuntimeError("libt2b200.so ABI version mismatch")
    _lib = L
    return L


SELFTEST_LIB_PATH = os.path.join(_HERE, "libt2b200_selftest.so")
SELFTEST_EXPORTS = ["t2_selftest_event", "t2_selftest_mma_rate", "t2_selftest_mma_group", "t2_selftest_gemm_tc", "t2_selftest_colsum",
                    "t2_selftest_waveglow_state"]
_selftest_lib = None


def selftest_lib():
    """libt2b200_selftest.so: the product sources built with -DT2_SELFTEST (adds t2_selftest_*); tests / tools only."""
    global _selftest_lib
    if _selftest_lib is None:
        if not os.path.isfile(SELFTEST_LIB_PATH):
            raise RuntimeError("tacotron2_b200: %s is missing -- run `make -C tacotron2_b200/csrc`" % SELFTEST_LIB_PATH)
        L = C.CDLL(SELFTEST_LIB_PATH)
        L.t2_last_error.restype = C.c_char_p
        L.t2_selftest_event.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_void_p]
        L.t2_selftest_mma_rate.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
        L.t2_selftest_mma_group.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
        L.t2_selftest_gemm_tc.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_float, C.c_int32, C.c_int64,
                                          C.c_int64, C.c_int64, C.c_void_p]
        L.t2_selftest_colsum.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
        L.t2_selftest_waveglow_state.argtypes = [C.c_void_p, C.POINTER(T2WaveGlowWindowArgs), C.c_int32] + [C.c_void_p] * 6
        L.t2_waveglow_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(T2WaveGlowConfig), C.POINTER(C.c_void_p),
                                         C.c_int32, C.c_void_p]
        L.t2_waveglow_destroy.argtypes = [C.c_void_p]
        L.t2_waveglow_workspace_bytes.restype = C.c_size_t
        L.t2_waveglow_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        _selftest_lib = L
    return _selftest_lib


def check_selftest(rc):
    if rc != 0:
        raise T2Error("libt2b200_selftest error %d: %s" % (rc, selftest_lib().t2_last_error().decode()))


class T2Error(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise T2Error("libt2b200 error %d: %s" % (rc, lib().t2_last_error().decode()))


def call(fn, device, *args):
    """fn(*args, stream) on `device`, where stream is torch's current CUDA stream there; raises T2Error on failure."""
    with torch.cuda.device(device):
        check(fn(*args, C.c_void_p(torch.cuda.current_stream(device).cuda_stream)))


def byte_buffer(nbytes, device):
    """An uninitialised device buffer of nbytes bytes (workspaces, stashes, stream state)."""
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


class Workspace:
    """Device workspaces by tag, reused while large enough.  A larger request or another device frees the old buffer
    before it allocates the new one, so the two never coexist."""

    def __init__(self):
        self._bufs = {}

    def get(self, tag, nbytes, device):
        t = self._bufs.get(tag)
        if t is None or t.numel() < nbytes or t.device != device:
            t = self._bufs[tag] = None
            t = self._bufs[tag] = byte_buffer(nbytes, device)
        return t

    def __getitem__(self, tag):
        return self._bufs[tag]
