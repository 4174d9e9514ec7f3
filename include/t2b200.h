/*
 * t2b200.h -- C ABI of libt2b200.so, the H100 (sm_90a) Tacotron 2 mel-spectrogram engine.
 *
 * The reference (NVIDIA/tacotron2) has no FFI / plugin layer: its hot path is ordinary Python
 * methods on nn.Modules (SURVEY.md section 8(b)).  This header is therefore the boundary a
 * maintainer of the reference would bind (ctypes stub in INTEGRATION.md) to replace, one for one,
 * the bodies of
 *
 *     Encoder.inference / Encoder.forward     model.py:173-201     -> t2_encoder_forward
 *     Decoder.inference                       model.py:418-454     -> t2_decoder_run (mode INFER)
 *     Decoder.forward  (teacher forcing)      model.py:381-416     -> t2_decoder_run (mode TEACHER)
 *       Prenet.forward                        model.py:97-100         (inside, per step / hoisted)
 *       Decoder.decode                        model.py:340-379        (inside, the persistent loop)
 *       Attention.forward / LocationLayer     model.py:22-26, 43-86   (inside)
 *       initialize_decoder_states             model.py:258-289        (inside: processed_memory GEMM)
 *     Decoder.decode, one step on caller state  model.py:340-379     -> t2_decoder_step
 *     Attention.forward / LocationLayer alone   model.py:22-26, 43-86 -> t2_attention_forward
 *     memory_layer(memory)                      model.py:288         -> t2_processed_memory
 *     Postnet.forward (+ residual add)        model.py:141-146, 511, 524  -> t2_postnet_forward
 *     Tacotron2.inference, host buffers       model.py:517-529     -> t2_infer_host
 *
 * Conventions
 *   - plain C types only; every tensor argument is a raw pointer into DEVICE memory of the current
 *     CUDA device unless its name ends in _host; all float tensors are fp32, contiguous;
 *   - the caller owns every buffer; the library allocates only inside T2Model (packed weights) and
 *     never frees caller memory; scratch comes from the caller-provided workspace (size queries);
 *   - a workspace, stash or stream state buffer needs no particular alignment: each call aligns its
 *     base itself, and the byte count its size query returns already includes that reserve, so a
 *     buffer of exactly that many bytes at any address is enough.  A stash is laid out the same way
 *     by the forward call that fills it and the backward call that reads it;
 *   - work is enqueued on the given stream (a cudaStream_t passed as void*); no call synchronises
 *     the device unless documented (t2_infer_host does, it returns host data);
 *   - every function returns 0 on success or a negative T2_ERR_* code; t2_last_error() returns a
 *     thread-local message for the last failure.  Nothing falls back to a CPU path.
 */
#ifndef T2B200_H_
#define T2B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define T2_ABI_VERSION 2

#define T2_OK               0
#define T2_ERR_INVALID     -1   /* bad argument / unsupported shape                     */
#define T2_ERR_CUDA        -2   /* a CUDA runtime call failed (message has the detail)  */
#define T2_ERR_WORKSPACE   -3   /* workspace too small                                  */
#define T2_ERR_UNSUPPORTED -4   /* hyper-parameters outside what the kernels implement  */
#define T2_ERR_WATCHDOG    -5   /* a device-side wait timed out (kernel aborted itself)  */

typedef struct T2Model T2Model; /* opaque: configuration + packed device-side weights */

/* Hyper-parameters the model code reads (hparams.py:40-75).  The kernels are specialised for the
 * reference defaults; t2_model_create returns T2_ERR_UNSUPPORTED for anything else. */
typedef struct T2Config {
  int32_t n_mel_channels;              /* 80   */
  int32_t n_symbols;                   /* 148  */
  int32_t symbols_embedding_dim;       /* 512  */
  int32_t encoder_kernel_size;         /* 5    */
  int32_t encoder_n_convolutions;      /* 3    */
  int32_t encoder_embedding_dim;       /* 512  */
  int32_t attention_rnn_dim;           /* 1024 */
  int32_t decoder_rnn_dim;             /* 1024 */
  int32_t prenet_dim;                  /* 256  */
  int32_t attention_dim;               /* 128  */
  int32_t attention_location_n_filters;    /* 32 */
  int32_t attention_location_kernel_size;  /* 31 */
  int32_t postnet_embedding_dim;       /* 512  */
  int32_t postnet_kernel_size;         /* 5    */
  int32_t postnet_n_convolutions;      /* 5    */
  float   p_attention_dropout;         /* 0.1  */
  float   p_decoder_dropout;           /* 0.1  */
  float   bn_eps;                      /* 1e-5 */
} T2Config;

/* Number of entries of the weight table: the reference state_dict in its own order
 * (84 tensors = 60 parameters + 24 BatchNorm buffers; SURVEY.md section 8(b1)). */
#define T2_NUM_WEIGHTS 84

/* Decoder implementations selectable at run time (both are CUDA; there is no CPU path). */
#define T2_IMPL_AUTO        0   /* persistent kernel when the shape allows, else STEPWISE */
#define T2_IMPL_STEPWISE    1   /* one fp32 kernel sequence per step (bring-up / cross-check) */
#define T2_IMPL_PERSISTENT  2   /* one persistent cooperative wgmma kernel for the whole loop */

#define T2_MODE_INFER    0      /* Decoder.inference: free running, prenet on the fed-back frame */
#define T2_MODE_TEACHER  1      /* Decoder.forward : teacher forced, exactly n_steps_cap steps  */

int         t2_abi_version(void);
const char* t2_last_error(void);

/* Fills {sm_count, cc_major, cc_minor, l2_bytes, max_smem_optin} of the current device. */
int t2_device_info(int32_t out[5]);

/* weights[i]: device pointer to the i-th state_dict tensor (fp32; the three int64
 * num_batches_tracked entries are ignored and may be NULL).  The model keeps the pointers (not
 * copies) of the fp32 tensors it streams directly and builds packed copies of the rest, so the
 * caller must re-create (or t2_model_refresh) the handle after the parameters change. */
int t2_model_create(T2Model** out, const T2Config* cfg, const void* const* weights,
                    int32_t n_weights, void* stream);
int t2_model_refresh(T2Model* m, const void* const* weights, int32_t n_weights, void* stream);
int t2_model_destroy(T2Model* m);

/* ---- Encoder (model.py:149-201) --------------------------------------------------------------
 * text (B, T) int64 symbol ids  ->  memory (B, T, 512).
 * lengths: NULL = Encoder.inference (every row full length); else (B) int32, sorted descending,
 * lengths[0] == T = Encoder.forward's packed-sequence semantics (zeros at padded positions).
 * training != 0: batch-statistics BatchNorm (+ running stat update into the caller's tensors)
 * and dropout(0.5) with keep masks (3, B, 512, T) uint8 or Philox(seed) when NULL. */
typedef struct T2EncoderArgs {
  const int64_t* text;                 /* (B, T) symbol ids, or NULL when `embedded` is given        */
  const float* embedded;               /* (B, T, 512) embedded inputs (model.py:503 before transpose) */
  const int32_t* lengths; int32_t B, T;
  int32_t training; const uint8_t* keep; uint64_t seed;
  float* memory;                       /* out (B, T, 512) */
  void* ws; size_t ws_bytes;
  void* stash; size_t stash_bytes;     /* optional: activations kept for t2_encoder_backward (any B; needs
                                          >= 128 SMs: the BiLSTM runs persistent, once per 64-row slice) */
} T2EncoderArgs;
size_t t2_encoder_workspace_bytes(const T2Model* m, int32_t B, int32_t T);
int    t2_encoder_forward(T2Model* m, const T2EncoderArgs* a, void* stream);
/* Encoder.inference over a batch of texts of different lengths: row b is encoded exactly as its first lengths[b]
 * symbols alone (a B = 1 call with T = lengths[b]), bit for bit.  lengths (B) int32, each in [1, T], in any order (not
 * checked here: the caller validates them); NULL = every row T long, the same as t2_encoder_forward without lengths.
 * Symbols at t >= lengths[b] are not read and memory there is zero.  Evaluation only: training must be 0 and stash
 * NULL (T2_ERR_INVALID otherwise).  Workspace: t2_encoder_workspace_bytes(m, B, T). */
int    t2_encoder_infer(T2Model* m, const T2EncoderArgs* a, void* stream);

/* Encoder backward (autograd graph of Encoder.forward, model.py:173-190): the stash of a forward call with the same
 * text / embedded, lengths, training, keep and seed; d_memory (B, T, 512) -> gradients of the encoder parameters
 * (grads[] entries that are non-NULL are overwritten; with `text` also embedding.weight) and, if non-NULL,
 * d_embedded (B, T, 512).  Any B: the BiLSTM's reverse recurrence runs per 64-row slice, the conv stack's backward
 * (BatchNorm over the whole batch) and the embedding gradient once.  The embedding gradient keeps the B x T symbol
 * ids in shared memory: B * T <= 51,200 (e.g. B = 128 at T = 400), else T2_ERR_UNSUPPORTED. */
typedef struct T2EncoderBwdArgs {
  const int64_t* text; const float* embedded; const int32_t* lengths; int32_t B, T;
  int32_t training; const uint8_t* keep; uint64_t seed;
  const void* stash; size_t stash_bytes;
  const float* d_memory;
  float* d_embedded;
  float* const* grads; int32_t n_grads;
  void* ws; size_t ws_bytes;
} T2EncoderBwdArgs;
size_t t2_encoder_stash_bytes(const T2Model* m, int32_t B, int32_t T);
size_t t2_encoder_backward_workspace_bytes(const T2Model* m, int32_t B, int32_t T);
int    t2_encoder_backward(T2Model* m, const T2EncoderBwdArgs* a, void* stream);

/* ---- Decoder (model.py:204-454) --------------------------------------------------------------
 * One call runs the whole autoregressive loop.
 *   memory (B, T_enc, 512); memory_lengths (B) int32 or NULL (no masking, model.py:432).
 *   INFER  : go frame -> [prenet -> decode -> stop test] x n; per-row stop latch
 *            done[b] |= sigmoid(gate[b]) > gate_threshold  (predicate of model.py:443);
 *            the loop ends when every row has fired or after n_steps_cap (= max_decoder_steps);
 *            rows that fired keep decoding, mel_lengths[b] = first firing step + 1.
 *   TEACHER: teacher_prenet (n_steps_cap, B, 256) = prenet outputs of go frame + targets
 *            (model.py:396-399); training != 0 applies dropout(p_att / p_dec) to the recurrent
 *            hidden states (model.py:355-356, 370-371) with att_keep / dec_keep
 *            (n_steps_cap, B, 1024) uint8 or Philox when NULL.
 *   prenet_keep: (n_steps_cap, 2, B, 256) uint8 keep masks for the always-on prenet dropout
 *            (model.py:99), or NULL => in-kernel Philox4x32-10 keyed by (seed, step).
 * Outputs (row-major): mel (B, T_cap, 80), gate (B, T_cap), align (B, T_cap, T_enc) where
 * T_cap = n_steps_cap; entries at t >= *n_steps are left untouched.  mel_lengths (B) int32,
 * n_steps (1) int32 on the device. */
/* In INFER mode every reduction over encoder positions of row b -- the masked softmax, the location filter near the
 * row's end, the context over staged and L2-resident memory rows -- runs in the order a call with T_enc =
 * memory_lengths[b] uses, so a row of a ragged batch equals its own B = 1 call on memory[b, :memory_lengths[b]] bit
 * for bit (persistent implementation; the stepwise one sums positions in a fixed order too). */
/* Per-row seeds (row_seeds != NULL; INFER, training = 0, prenet_keep NULL -- T2_ERR_INVALID otherwise): row b draws
 * the prenet keep bit of its step s, layer k, column j as Philox keyed by (row_seeds[b], site 4 s + k, element j), which
 * is what a B = 1 call with seed = row_seeds[b] draws.  Row b's outputs then equal that call's bit for bit, whatever
 * its batch, its 64-row slice, the stream chunking or the serving slot.  NULL: one key for the call, element
 * b * 256 + j. */
/* Forced alignment (forced_align and forced_lengths both set; INFER, training = 0, persistent implementation): the
 * attention weights are given instead of computed, as in Mellotron's inference_noattention.  forced_align
 * (B, n_steps_cap, T_enc) fp32 and forced_lengths (B) int32 are on the device.  Row b runs forced_lengths[b] steps (the
 * call clamps each into [1, n_steps_cap] and never reads outside the map); at step t < forced_lengths[b] its context is
 * sum_j forced_align[b, t, j] * memory[b, j] over j < memory_lengths[b] -- the weights are used as given, not normalised
 * or checked -- and every other step of the row (its 64-row slice is still running) uses zero weights.  align holds
 * the weights used: the given ones below memory_lengths[b], zero beyond.  The gate is computed and written but stops
 * nothing, and gate_threshold plays no part: mel_lengths[b] = forced_lengths[b], and the loop ends when every row has
 * run its steps.  The prenet, both LSTMs, the projection and the dropout keys are those of the free run, so feeding a
 * free run's own align and mel_lengths back reproduces its mel and gate bit for bit.  Both NULL: today's behaviour.
 * T2_ERR_INVALID: only one of the two set, mode TEACHER, or training = 1; T2_ERR_UNSUPPORTED: the stepwise
 * implementation (requested, or chosen by AUTO for a T_enc the persistent kernel does not take).  The resumable
 * stream indexes the map by absolute step; continuous batching (admit / collect) and t2_infer_host take no map. */
typedef struct T2DecoderArgs {
  int32_t mode, impl, training;
  const float* memory; const int32_t* memory_lengths; int32_t B, T_enc, n_steps_cap;
  const float* teacher_prenet;
  const uint8_t* prenet_keep; const uint8_t* att_keep; const uint8_t* dec_keep;
  uint64_t seed;
  float gate_threshold, score_mask_value;
  float* mel; float* gate; float* align; int32_t* mel_lengths; int32_t* n_steps;
  void* ws; size_t ws_bytes;
  void* stash; size_t stash_bytes;     /* TEACHER only, optional: activations kept for t2_decoder_backward
                                          (t2_decoder_stash_bytes(); opaque to the caller) */
  const uint64_t* row_seeds;           /* (B) or NULL: per-row Philox keys of the prenet dropout (see below) */
  const float* forced_align;           /* (B, n_steps_cap, T_enc) or NULL: given attention weights (see above) */
  const int32_t* forced_lengths;       /* (B) or NULL: steps of each row of a forced run */
  int32_t window_back, window_front;   /* 0, 0: no attention window (see below) */
  const int32_t* max_steps;            /* (B) or NULL: each row's step limit (see below) */
} T2DecoderArgs;
size_t t2_decoder_workspace_bytes(const T2Model* m, int32_t B, int32_t T_enc, int32_t n_steps_cap);
int    t2_decoder_run(T2Model* m, const T2DecoderArgs* a, void* stream);
/* Limits (INFER, persistent implementation): guards for free runs whose attention may jump, repeat or never reach the
 * end of the text.  They are set when window_front != 0, window_back != 0 or max_steps != NULL; a zeroed struct sets none.
 *   window_back, window_front: an attention window (ESPnet's use_att_constraint with backward / forward window).  Let
 *     p_t(b) be the smallest j < memory_lengths[b] that maximises row b's weights of step t - 1 (0 at step 0, and at the
 *     first step of a row put back by admit, whose weights are all zero).  At step t the energies of row b at
 *     j < p_t - window_back and at j >= p_t + window_front get score_mask_value before the softmax, on top of the length
 *     mask, so the weights outside [p_t - window_back, p_t + window_front) come out 0.  Everything else -- the location
 *     term (from these weights), the context, both LSTMs, the gate and the dropout keys -- is the free run's.  p_t comes
 *     from the previous weights, which a stream already saves, so streams and continuous batching need no extra state.
 *     window_front = 0 (with window_back = 0): no window.  A window with both sides >= memory_lengths[b] masks nothing
 *     and gives the unwindowed bits.
 *   max_steps: (B) int32 on the device, or NULL: row b also stops after max_steps[b] steps (clamped into
 *     [1, n_steps_cap] where read) if its gate has not fired before; mel_lengths[b] is then max_steps[b].  The loop ends
 *     when every row has stopped, so n_steps_cap = the largest limit wastes no steps on rows that reached theirs.
 * Row b then equals bit for bit its own B = 1 call with n_steps_cap = max_steps[b] and the same window.
 * T2_ERR_INVALID: limits with forced_align, mode TEACHER, a negative window side, or window_back != 0 without a window;
 * T2_ERR_UNSUPPORTED: the stepwise implementation (requested, or chosen by AUTO for a T_enc the persistent kernel does
 * not take).  t2_infer_host takes no limits. */

/* ---- One decoder step on the caller's state (Decoder.decode, model.py:340-379) ---------------------------------
 * For hand-written decoder loops (tacotron2_b200: Decoder.initialize_decoder_states / decode).  One call runs the step
 * after the prenet -- attention LSTM, attention, decoder LSTM, projection and gate -- on state arrays the caller holds,
 * with the stepwise implementation's kernels and arithmetic: the step of decoder_run_stepwise's loop, bit for bit.
 *   memory (B, T_enc, 512), processed_memory (B, T_enc, 128) (t2_processed_memory), mask (B, T_enc) uint8 or NULL:
 *   1 = padded position, whose energy gets score_mask_value before the softmax (model.py:79-80), any pattern.
 *   attention_hidden / attention_cell / decoder_hidden / decoder_cell (B, 1024), attention_weights /
 *   attention_weights_cum (B, T_enc), attention_context (B, 512): read and updated in place.
 *   decoder_input (B, 256): the prenet output.  mel (B, 80) and gate (B) out.
 *   training != 0: dropout(p_attention_dropout / p_decoder_dropout) on the two hidden states (model.py:355-356,
 *   370-371) with att_keep / dec_keep (B, 1024) uint8 keep masks, or NULL => Philox(seed) at the sites of step 0 of a
 *   t2_decoder_run, so one call equals that run's first step.
 * Every array starts on a 16-byte boundary (the GEMMs read rows as float4).
 * 7 kernel launches, no host synchronisation, no allocation.  T2_ERR_INVALID for null or misaligned pointers, B outside [1, 1024],
 * T_enc < 1 or too small a workspace (t2_decoder_step_workspace_bytes(m, B)); T2_ERR_UNSUPPORTED for T_enc > 1282 (the
 * stepwise attention's shared memory); both before any launch. */
typedef struct T2DecoderStepArgs {
  int32_t B, T_enc;
  const float* memory; const float* processed_memory; const uint8_t* mask;
  float* attention_hidden; float* attention_cell; float* decoder_hidden; float* decoder_cell;
  float* attention_weights; float* attention_weights_cum; float* attention_context;
  const float* decoder_input;
  float* mel; float* gate;
  int32_t training; const uint8_t* att_keep; const uint8_t* dec_keep; uint64_t seed;
  float score_mask_value;
  void* ws; size_t ws_bytes;
} T2DecoderStepArgs;
size_t t2_decoder_step_workspace_bytes(const T2Model* m, int32_t B);
int    t2_decoder_step(T2Model* m, const T2DecoderStepArgs* a, void* stream);

/* Attention.forward, Attention.get_alignment_energies and LocationLayer.forward (model.py:22-26, 43-86) in one launch
 * of the step's attention kernel.  attention_weights_cat (B, 2, T_enc): previous and cumulative weights, as given.
 * query (B, 1024) and processed_memory (B, T_enc, 128) may be NULL (zero) when only `location` is wanted; memory
 * (B, T_enc, 512) is read only for `context`; mask as for t2_decoder_step.  Outputs, each optional: energies (B, T_enc)
 * before masking, location (B, T_enc, 128) the location term, weights (B, T_enc) the masked softmax, context (B, 512).
 * No cumulative array is touched.  With the inputs of a t2_decoder_step, weights and context are that step's bit for
 * bit.  Refusals as t2_decoder_step (at least one output, context needs memory, weights or context need query and
 * processed_memory). */
typedef struct T2AttentionArgs {
  int32_t B, T_enc;
  const float* query; const float* memory; const float* processed_memory; const float* attention_weights_cat;
  const uint8_t* mask;
  float score_mask_value;
  float* energies; float* location; float* weights; float* context;
} T2AttentionArgs;
int    t2_attention_forward(T2Model* m, const T2AttentionArgs* a, void* stream);

/* memory_layer(memory) (model.py:288): memory (B, T_enc, 512), 16-byte aligned -> out (B, T_enc, 128), the GEMM the stepwise decoder
 * uses, so t2_decoder_step on it computes what t2_decoder_run (STEPWISE) computes. */
int    t2_processed_memory(T2Model* m, const float* memory, int32_t B, int32_t T_enc, float* out, void* stream);

/* ---- Resumable decoder stream: the INFER loop of t2_decoder_run in chunks of steps -------------
 * The same persistent kernel stops after a number of steps and resumes exactly where it stopped, so
 * the steps of all chunks together compute bit for bit what one t2_decoder_run computes (dropout is
 * keyed by the absolute step).  Everything that lives across a step boundary is kept in the caller's
 * `state` buffer (t2_decoder_stream_state_bytes), one block per 64-row slice: several streams can be
 * alive on one model at a time, and t2_decoder_run's workspace is not used.
 *   dec: as for t2_decoder_run with mode = INFER (teacher_prenet, att_keep, dec_keep, ws and stash are
 *        not used; memory_lengths is, as by t2_decoder_run).  The limits apply to every chunk; dec.max_steps count
 *        absolute steps, so admit refuses a stream that carries them (T2_ERR_INVALID).  mel / gate / align are the full
 *        n_steps_cap-sized buffers; each run writes its steps at their absolute indices.  mel_lengths[b] =
 *        -1 while row b is live, then its length, as t2_decoder_run.  T2_IMPL_STEPWISE and encoder
 *        lengths the persistent kernel does not take are refused with T2_ERR_UNSUPPORTED.
 *   status: device int32 (2 x ceil(B / 64)): [steps run, stopped] per slice, written by every run.
 * begin zeroes the state, sets mel_lengths to -1 and computes the processed memory; it does not
 * touch mel / gate / align (zero them first, as for t2_decoder_run).  run advances every slice that
 * has not stopped by up to n_steps steps (one launch per slice, no host synchronisation);
 * status_host is the caller's copy of `status` after the previous run (NULL after begin): slices it
 * marks stopped are not launched again. */
typedef struct T2DecoderStreamArgs {
  T2DecoderArgs dec;
  void* state; size_t state_bytes;
  int32_t* status;
  const int32_t* row_step0;            /* (B) device or NULL: with dec.row_seeds, row b's step (the one its prenet keys
                                          use) at local step i of a run is row_step0[b] + i instead of the absolute step */
} T2DecoderStreamArgs;
size_t t2_decoder_stream_state_bytes(const T2Model* m, int32_t B, int32_t T_enc);
int    t2_decoder_stream_begin(T2Model* m, const T2DecoderStreamArgs* a, void* stream);
int    t2_decoder_stream_run(T2Model* m, const T2DecoderStreamArgs* a, int32_t n_steps, const int32_t* status_host,
                             void* stream);

/* ---- Continuous batching on a decoder stream: its rows as slots ---------------------------------
 * A row's bits depend neither on its neighbours nor on T_enc, and between two runs all of its state is
 * in `state`, so a row can be handed another text there.  Such a session runs every chunk as local
 * steps [0, n): t2_decoder_stream_run with status_host = NULL (every slice starts at step 0; a
 * status_host of [0, 1] pairs skips slices) on a stream whose n_steps_cap is n + 1 -- the kernel keeps
 * no step counter in `state`, and a step reads the keep mask of the step after it.  mel / gate / align
 * are chunk buffers (B, n + 1, .), prenet_keep (n + 1, 2, B, 256) holds at [i, :, b] the mask of row b's
 * own step (steps it has run before the chunk) + i, and dec.seed is the chunk's Philox seed; the caller
 * rewrites them (and memory / memory_lengths rows) between runs.  Seeded instead (dec.row_seeds, prenet_keep NULL):
 * row_step0[b] holds the steps row b's request has run before the chunk, and each request draws its own B = 1 stream.  mel_lengths[b] becomes the local step
 * + 1 at which row b fired in the chunk; a slice ends a chunk early once all its rows have fired.
 *   admit:   rows (host, n_rows ascending row indices): each listed row goes back to the state begin
 *            gives it -- its accumulator rows, LSTM cells, previous / cumulative attention weights,
 *            rows of the activation images and of the query, stop latch, mel_lengths[row] = -1 -- and
 *            its processed memory is recomputed from memory[row] (one reset launch whatever n_rows is,
 *            and one GEMM per run of consecutive rows).  No other row's state is written.
 *   collect: rows (host): the first n_frames frames of chunk row `row` -- mel, gate and
 *            align[:, :T_text] -- are copied to mel (n_frames, 80), gate (n_frames), align (n_frames,
 *            T_text) of the entry: the request's own buffers at its own step offset.  One launch per
 *            64-row slice with entries.
 * Both refuse rows outside [0, B), counts outside the chunk buffers and null pointers before any launch. */
typedef struct T2CollectRow {
  int32_t row, n_frames, T_text, reserved;
  float* mel; float* gate; float* align;
} T2CollectRow;
int    t2_decoder_stream_admit(T2Model* m, const T2DecoderStreamArgs* a, const int32_t* rows, int32_t n_rows, void* stream);
int    t2_decoder_stream_collect(T2Model* m, const T2DecoderStreamArgs* a, const T2CollectRow* rows, int32_t n_rows,
                                 void* stream);

/* ---- Decoder backward (the autograd graph of Decoder.forward, model.py:381-416) ----------------
 * Reverse-time recurrence over the stash of a TEACHER run with the same memory / teacher_prenet / masks /
 * seed, then the time-batched weight gradients.  Any B >= 1: the recurrence runs its 64-row slices side by side
 * (a row's phase-1 results do not depend on its slice), the weight gradients take all T_mel x B rows at once.
 *   d_mel (B, T_mel, 80), d_gate (B, T_mel): gradients wrt the mel / gate outputs (same layout as the
 *   outputs); d_align (B, T_mel, T_enc) or NULL.
 *   d_memory (B, T_enc, 512) and d_prenet (T_mel, B, 256) (gradient wrt teacher_prenet) are written.
 *   grads: T2_NUM_WEIGHTS pointers in state_dict order; the decoder entries that are non-NULL (attention_rnn,
 *   attention_layer, decoder_rnn, linear_projection, gate_layer) are OVERWRITTEN with the gradient of the
 *   corresponding parameter.  The prenet parameters are handled by t2_prenet_backward. */
typedef struct T2DecoderBwdArgs {
  const float* memory; const int32_t* memory_lengths; int32_t B, T_enc, T_mel;
  int32_t training;                    /* same value as the forward call (hidden-state dropout on / off) */
  const float* teacher_prenet;
  const uint8_t* att_keep; const uint8_t* dec_keep; uint64_t seed;
  float score_mask_value;
  const float* align;                  /* (B, T_mel, T_enc) forward output */
  const void* stash; size_t stash_bytes;
  const float* d_mel; const float* d_gate; const float* d_align;
  float* d_memory; float* d_prenet;
  float* const* grads; int32_t n_grads;
  void* ws; size_t ws_bytes;
} T2DecoderBwdArgs;
size_t t2_decoder_stash_bytes(const T2Model* m, int32_t B, int32_t T_enc, int32_t T_mel);
size_t t2_decoder_backward_workspace_bytes(const T2Model* m, int32_t B, int32_t T_enc, int32_t T_mel);
int    t2_decoder_backward(T2Model* m, const T2DecoderBwdArgs* a, void* stream);

/* Backward of t2_prenet_forward: frames (M, 80), the same keep / seed, d_out (M, 256) ->
 * grads[prenet.layers.0 / 1] overwritten (d_frames is not needed: the frames are data, model.py:396-399). */
typedef struct T2PrenetBwdArgs {
  const float* frames; int32_t M; const uint8_t* keep; uint64_t seed;
  const float* d_out;
  float* const* grads; int32_t n_grads;
  void* ws; size_t ws_bytes;
} T2PrenetBwdArgs;
size_t t2_prenet_backward_workspace_bytes(const T2Model* m, int32_t M);
int    t2_prenet_backward(T2Model* m, const T2PrenetBwdArgs* a, void* stream);

/* Prenet over a block of frames (teacher forcing hoists it out of the loop, model.py:399):
 * frames (M, 80) -> out (M, 256); keep (2, M, 256) uint8 or NULL => Philox(seed). */
int t2_prenet_forward(T2Model* m, const float* frames, int32_t M, const uint8_t* keep,
                      uint64_t seed, float* out, void* ws, size_t ws_bytes, void* stream);

/* ---- Postnet (model.py:103-146) + residual (model.py:511 / 524) ------------------------------
 * mel (B, T, 80) time-major per row (the decoder's native storage; the reference's (B,80,T)
 * tensor is a transposed view of exactly this, model.py:336)  ->  mel_post (B, 80, T) contiguous
 * = mel^T + postnet(mel^T).  lengths (B) int32 or NULL: frames t >= lengths[b] of the INPUT are
 * treated as zero and the output there is zero (batched-inference padding, see README). */
typedef struct T2PostnetArgs {
  const float* mel;
  int64_t mel_batch_stride;            /* elements between rows b and b+1 of mel; 0 = T*80 */
  const int32_t* lengths; int32_t B, T;
  int32_t training; const uint8_t* keep; uint64_t seed;
  int32_t add_residual;                /* 1: mel_post = mel^T + postnet(mel^T) (model.py:511, 524); 0: postnet only */
  float* mel_post;
  void* ws; size_t ws_bytes;
  void* stash; size_t stash_bytes;     /* optional (lengths must be NULL): activations kept for t2_postnet_backward */
} T2PostnetArgs;
size_t t2_postnet_workspace_bytes(const T2Model* m, int32_t B, int32_t T);
int    t2_postnet_forward(T2Model* m, const T2PostnetArgs* a, void* stream);
/* The postnet of a ragged inference batch: as t2_postnet_forward, but row b is computed exactly as its first lengths[b]
 * frames alone (a B = 1 call with T = lengths[b]), bit for bit -- every hidden layer is zero at t >= lengths[b] too, the
 * padding each convolution sees at that length, where t2_postnet_forward runs the hidden layers over the zero frames.
 * lengths NULL: the same as t2_postnet_forward.  Evaluation only: training must be 0 and stash NULL. */
int    t2_postnet_infer(T2Model* m, const T2PostnetArgs* a, void* stream);

/* Postnet backward (model.py:141-146 + the residual of :511): d_mel_post (B, 80, T) -> d_mel (B, T, 80) (gradient wrt
 * the input rows, including the residual branch when add_residual) and the postnet parameter gradients. */
typedef struct T2PostnetBwdArgs {
  int32_t B, T, training, add_residual; const uint8_t* keep; uint64_t seed;
  const int32_t* wgrad_lengths;        /* (B) or NULL: frames t >= wgrad_lengths[b] of the stashed INPUT count as zero in the
                                          first conv's weight gradient -- what the reference's autograd computes, because
                                          parse_output zeroes that tensor in place after the forward pass (model.py:492) */
  const void* stash; size_t stash_bytes;
  const float* d_mel_post;
  float* d_mel;
  float* const* grads; int32_t n_grads;
  void* ws; size_t ws_bytes;
} T2PostnetBwdArgs;
size_t t2_postnet_stash_bytes(const T2Model* m, int32_t B, int32_t T);
size_t t2_postnet_backward_workspace_bytes(const T2Model* m, int32_t B, int32_t T);
int    t2_postnet_backward(T2Model* m, const T2PostnetBwdArgs* a, void* stream);

/* ---- Fused gradient clipping + Adam (train.py:229-236: clip_grad_norm_ then torch.optim.Adam.step) -----------
 * n tensors (host arrays of device pointers + element counts).  grad_norm (device, 1 float) receives the total
 * gradient norm BEFORE clipping; the gradients are scaled in place by min(1, max_norm / (norm + 1e-6)) like
 * torch.nn.utils.clip_grad_norm_ (max_norm <= 0: no clipping), then exp_avg / exp_avg_sq / the parameters are updated
 * exactly like torch.optim.Adam (L2 weight decay, bias correction with `step` counted from 1). */
typedef struct T2AdamArgs {
  int32_t n;
  float* const* params; float* const* grads; float* const* exp_avg; float* const* exp_avg_sq; const int64_t* numel;
  double lr, beta1, beta2, eps, weight_decay, max_norm;   /* doubles: 1 - beta2^step must not be rounded through fp32 */
  int32_t step;
  float* grad_norm;
  void* ws; size_t ws_bytes;
} T2AdamArgs;
size_t t2_clip_adam_workspace_bytes(int64_t total_elements, int32_t n_tensors);
int    t2_clip_adam_step(const T2AdamArgs* a, void* stream);

/* ---- mixed-precision optimizer step (the reference trains "fp16" through Apex AMP O2, train.py:173-176, 222-236) ------
 * fp16 (or fp32) model parameters + fp32 master copies; gradients arrive in the parameter's dtype multiplied by the
 * dynamic loss scale state[0].  One call = unscale, overflow check, clip_grad_norm_ on the unscaled gradients, Adam on
 * the masters, write-back of the model copies, loss-scaler update (apex LossScaler: overflow -> skip the step, scale *
 * backoff_factor; growth_interval consecutive good steps -> scale * growth_factor).  Three multi-tensor launches, no host
 * synchronisation: `state` (4 floats on the device: loss scale, good steps since the last scale change, optimizer steps
 * taken -- skipped steps do not count --, 1.0 if this step was skipped) carries everything between calls. */
typedef struct T2AmpAdamArgs {
  int32_t n;
  void* const* model_params; const int32_t* param_is_half;   /* per tensor: storage read by the model, 1 = __half */
  const void* const* grads;  const int32_t* grad_is_half;    /* per tensor: gradient x loss scale */
  float* const* master; float* const* exp_avg; float* const* exp_avg_sq; const int64_t* numel;
  double lr, beta1, beta2, eps, weight_decay, max_norm;
  int32_t growth_interval; float growth_factor, backoff_factor;
  float* state;            /* device, 4 floats (see above) */
  float* grad_norm;        /* device out: norm of the unscaled gradients before clipping (inf / nan on overflow) */
  int32_t* skipped;        /* device out (may be NULL): 1 = overflow, nothing was updated */
  void* ws; size_t ws_bytes;
} T2AmpAdamArgs;
size_t t2_amp_adam_workspace_bytes(int64_t total_elements, int32_t n_tensors);
int    t2_amp_adam_step(const T2AmpAdamArgs* a, void* stream);

/* ---- Tacotron2Loss fused with the parse_output mask and the gradient seeds (loss_function.py:8-19, model.py:487-497) ----
 * mel / mel_post (B, C, T) contiguous fp32, gate (B, T), targets of the same shapes.  output_lengths (B) int32 or NULL: when
 * given, frames t >= output_lengths[b] of mel / mel_post are zeroed and of gate set to 1e3 IN PLACE before they enter the
 * loss (parse_output).  loss[0] = MSE(mel) + MSE(mel_post) + BCEWithLogits(gate), loss[1..3] the three terms.  d_mel /
 * d_mel_post / d_gate (each may be NULL): d loss / d output, written in the same pass. */
typedef struct T2LossArgs {
  float* mel; float* mel_post; float* gate;
  const float* mel_target; const float* gate_target;
  const int32_t* output_lengths;
  int32_t B, C, T;
  float* loss;                                   /* device, 4 floats */
  float* d_mel; float* d_mel_post; float* d_gate;
  void* ws; size_t ws_bytes;
} T2LossArgs;
size_t t2_loss_workspace_bytes(void);
int    t2_tacotron2_loss(const T2LossArgs* a, void* stream);

/* ---- TacotronSTFT.mel_spectrogram (layers.py:63-80, stft.py:69-94): batch of waveforms -> log-mel spectrograms ----------
 * y (B, n_samples) fp32 in [-1, 1] (not checked here; the Python mirror asserts it like the reference does).
 * forward_basis (2 * (filter_length / 2 + 1), filter_length): the windowed Fourier basis of stft.py:44-63;
 * mel_basis (n_mel, filter_length / 2 + 1).  mel out: (B, n_mel, n_frames) = log(max(mel_basis . |STFT|, clip_val)),
 * n_frames = n_samples / hop_length + 1 (reflect padding by filter_length / 2 on both sides).
 * lengths (device, B int32 sample counts, or NULL): row b is computed as y[b, :lengths[b]] alone -- bit for bit the B = 1
 * call on those samples -- and its frames from lengths[b] / hop_length + 1 on are zero; samples at or past lengths[b] are
 * never read.  Each length must lie in [filter_length / 2 + 1, n_samples]: the values live on the device, so the call
 * cannot refuse them without waiting for the GPU; the device clamps them into that range (the Python mirror refuses
 * them).  The workspace is t2_mel_spectrogram_workspace_bytes_lengths(B, n_samples, ...).  NULL: the whole batch shares
 * each frame's operand scale and its GEMM split plan, as before lengths existed. */
typedef struct T2MelSpecArgs {
  const float* y; int32_t B, n_samples;
  int32_t filter_length, hop_length, n_mel;
  const float* forward_basis; const float* mel_basis;
  float clip_val;
  float* mel;
  void* ws; size_t ws_bytes;
  const int32_t* lengths;
} T2MelSpecArgs;
int32_t t2_mel_spectrogram_frames(int32_t n_samples, int32_t hop_length);
size_t  t2_mel_spectrogram_workspace_bytes(int32_t B, int32_t n_samples, int32_t filter_length, int32_t hop_length, int32_t n_mel);
size_t  t2_mel_spectrogram_workspace_bytes_lengths(int32_t B, int32_t n_max, int32_t filter_length, int32_t hop_length,
                                                   int32_t n_mel);
int     t2_mel_spectrogram(const T2MelSpecArgs* a, void* stream);

/* ---- TextMelCollate on the device (data_utils.py:73-111): ragged batch in HBM -> the padded, length-sorted 5-tuple ------------
 * text_flat: the B token sequences concatenated (int64), text_offsets (B + 1) their prefix offsets; mel_flat: the B
 * (n_mel, L_i) row-major spectrograms concatenated, mel_offsets (B + 1) prefix offsets in FRAMES.  T_max >= longest text,
 * L_pad >= longest mel (the caller rounds it up to a multiple of n_frames_per_step, data_utils.py:93-96).  Rows are ordered by
 * decreasing text length (ties keep the original order); order[b] = source row of output row b.  All pointers device. */
typedef struct T2CollateArgs {
  const int64_t* text_flat; const int64_t* text_offsets;
  const float* mel_flat; const int64_t* mel_offsets;
  int32_t B, n_mel, T_max, L_pad;
  int32_t* order;
  int64_t* text_padded; int64_t* input_lengths;
  float* mel_padded; float* gate_padded; int64_t* output_lengths;
} T2CollateArgs;
int t2_collate(const T2CollateArgs* a, void* stream);

/* ---- Tacotron2.inference end to end with HOST buffers (model.py:517-529) ----------------------
 * text_host (B, T_text) int64 in (pinned) host memory -> mel_post_host (B, 80, max_steps) fp32,
 * mel_lengths_host (B), n_steps_host (1).  Copies H2D, runs encoder -> decoder -> postnet on
 * `stream`, copies D2H and synchronises the stream.  The postnet runs over the n_steps decoded
 * frames, as Tacotron2.inference does (so frames [0, n_steps) equal its mel_outputs_postnet); frames
 * beyond each row's length are zero.  Seed: the decoder's prenet dropout.  ws is device memory of
 * t2_infer_workspace_bytes().
 * Texts of different lengths: input_lengths_host (B) int64 in (pinned) host memory, each in [1, T_text], any order, or
 * NULL (every row T_text long).  Row b's outputs then equal those of a call on text_host[b, :input_lengths_host[b]]
 * alone (B = 1, same seed and impl) bit for bit, up to that call's n_steps; the ids at t >= input_lengths_host[b] are
 * ignored.  When every length is T_text the outputs are those of input_lengths_host = NULL (an equal-length batch keeps
 * its batched postnet, see t2_postnet_infer).  A length outside [1, T_text] is T2_ERR_INVALID before anything is
 * enqueued.  row_seeds_host needs input_lengths_host (T2_ERR_INVALID otherwise). */
typedef struct T2InferArgs {
  const int64_t* text_host;            /* (B, T_text) */
  const int64_t* input_lengths_host;   /* (B) or NULL */
  int32_t B, T_text, max_steps;
  float gate_threshold;
  uint64_t seed;
  int32_t impl;
  float* mel_post_host;                /* out (B, 80, max_steps) */
  int32_t* mel_lengths_host;           /* out (B) */
  int32_t* n_steps_host;               /* out (1) */
  void* ws; size_t ws_bytes;
  const uint64_t* row_seeds_host;      /* (B) host or NULL: the decoder's row_seeds (row b then equals its B = 1 call
                                          with seed = row_seeds_host[b]); `seed` is not used when given */
} T2InferArgs;
size_t t2_infer_workspace_bytes(const T2Model* m, int32_t B, int32_t T_text, int32_t max_steps);
int    t2_infer_host(T2Model* m, const T2InferArgs* a, void* stream);

/* ---- Durations from attention maps (tacotron2_b200.durations_from_alignments; DESIGN section 6.10) ----------------
 * alignments (B, T_mel, T_text) fp32 row-major -> durations (B, T_text) int64, frames per symbol.  Row b reads only
 * alignments[b, :L_mel, :L_text] (L_mel = mel_lengths[b], L_text = input_lengths[b]; a NULL array means T_mel / T_text
 * for every row) and writes zeros from L_text on, so it equals its own B = 1 call on that slice.  The lengths live on the
 * device: the call cannot refuse them without waiting for the GPU, so the device clamps them into [1, T_mel] /
 * [1, T_text] (the Python mirror refuses them).  Weights must be finite and >= 0 (not checked here; the Python mirror
 * does).
 *   T2_DURATIONS_MAS: the monotonic path from (0, 0) to (L_mel - 1, L_text - 1) -- per frame it stays on its symbol or
 *     advances by one -- that maximises the sum of log(max(a, 2^-126)), computed in fp64.  S[0][0] = c[0][0],
 *     S[0][j > 0] = -inf, S[t][j] = c[t][j] + max(S[t-1][j], S[t-1][j-1]); the backtrack from j = L_text - 1 at
 *     t = L_mel - 1 gives frame t to j and steps to j - 1 when j > 0 and (j == t or S[t-1][j-1] > S[t-1][j]), so ties
 *     stay on the current symbol.  Every symbol gets at least one frame; a row with L_mel < L_text has no such path and
 *     gets zeros.
 *   T2_DURATIONS_ARGMAX: frame t < L_mel goes to the smallest j < L_text holding the frame's maximum over j < L_text;
 *     a symbol may get 0 frames.
 * T_text <= T2_DURATIONS_MAX_TEXT (one CTA of at most 256 threads holds a row's scores, 16 symbols per thread).
 * Bad sizes, a bad method or a NULL alignments / durations / ws are T2_ERR_INVALID, too small a workspace
 * T2_ERR_WORKSPACE, before anything is launched.  No handle, no allocation, no host synchronisation.
 * Workspace: t2_durations_workspace_bytes(B, T_mel, T_text, method) (0 for arguments the call refuses). */
#define T2_DURATIONS_MAS       0
#define T2_DURATIONS_ARGMAX    1
#define T2_DURATIONS_MAX_TEXT  4096
typedef struct T2DurationsArgs {
  const float* alignments;             /* (B, T_mel, T_text) */
  const int32_t* input_lengths;        /* (B) device or NULL */
  const int32_t* mel_lengths;          /* (B) device or NULL */
  int32_t B, T_mel, T_text, method;
  int64_t* durations;                  /* out (B, T_text) */
  void* ws; size_t ws_bytes;
} T2DurationsArgs;
size_t t2_durations_workspace_bytes(int32_t B, int32_t T_mel, int32_t T_text, int32_t method);
int    t2_durations(const T2DurationsArgs* a, void* stream);

/* ---- Pitch targets (tacotron2_b200.pyin / average_by_durations; DESIGN section 6.11) ------------------------------
 * pYIN as librosa 0.10 computes it with center=True, pad_mode="constant", in fp64: y (B, n) fp32 row-major -> f0,
 * voiced_flag and voiced_prob, each (B, F) with F = 1 + n / hop_length (the frame count of t2_mel_spectrogram at
 * hop 256).  Row b reads only y[b, :L] (L = lengths[b]; a NULL array means n for every row), zero-pads it by
 * frame_length / 2 on both sides and has 1 + L / hop_length frames, so it equals its own B = 1 call; its later frames
 * get f0 0, voiced_flag 0 and voiced_prob 0.  Device lengths are clamped into [1, n] (the Python mirror refuses them).
 * Samples must be finite (not checked here; the Python mirror does).
 * The parameters arrive derived, as the host computes them from librosa's (tacotron2_b200.pitch.pyin_tables):
 *   min_period = floor(sr / fmax), max_period = min(ceil(sr / fmin), frame_length - win_length - 1) > min_period;
 *   n_bins = floor(12 bins_per_semitone log2(fmax / fmin)) + 1 <= T2_PYIN_MAX_BINS (the Viterbi CTA keeps 136 bytes
 *   per bin in shared memory); width = the local-triangle transition width, h = width / 2;
 *   thresholds[k] = linspace(0, 1, n_thresholds + 1)[k + 1], beta_probs = diff(beta.cdf(thresholds)),
 *   beta_prefix[m] = numpy sum(beta_probs[:m]) (m = 0..n_thresholds);
 *   boltzmann[N (N - 1) / 2 + p] = boltzmann.pmf(p, boltzmann_parameter, N) for N = 1..(max_period - min_period + 2) / 2,
 *   p < N;
 *   log_trans (2, 2h + 1, n_bins): [s][k][j] = log(T + tiny) of the transition from bin j - h + k to bin j within a
 *   voicing half (s = 0) or across (s = 1), T = kron(transition_loop(2, 1 - switch_prob), transition_local(n_bins,
 *   width, "triangle")); out of the band every entry is log(tiny) = log_tiny;
 *   log_init_unvoiced = log(1 / n_bins + tiny); freqs[k] = fmin 2^(k / (12 bins_per_semitone)).
 * f0 is freqs[state] on voiced frames and fill_na on unvoiced ones.  The decoded path equals the dense Viterbi's
 * (numpy argmax ties: the smallest index).  Bad sizes or a NULL pointer are T2_ERR_INVALID, too small a workspace
 * T2_ERR_WORKSPACE, before anything is launched.  2 launches, no handle, no allocation, no host synchronisation.
 * Workspace: t2_pyin_workspace_bytes(a) (reads only the sizes; 0 for arguments the call refuses): per frame
 * 4 n_bins + 10 ceil(lags / 2) + 12 bytes, lags = max_period - min_period + 1. */
#define T2_PYIN_MAX_FRAME       2048
#define T2_PYIN_MAX_BINS        1536
#define T2_PYIN_MAX_THRESHOLDS  4096
typedef struct T2PyinArgs {
  const float* y;                      /* (B, n) */
  const int32_t* lengths;              /* (B) device or NULL: samples per row */
  int32_t B, n, sr, frame_length, win_length, hop_length;
  int32_t min_period, max_period, n_thresholds, n_bins, bins_per_semitone, width;
  double fmin, no_trough_prob, fill_na, log_tiny, log_init_unvoiced;
  const double* thresholds;            /* (n_thresholds) */
  const double* beta_probs;            /* (n_thresholds) */
  const double* beta_prefix;           /* (n_thresholds + 1) */
  const double* boltzmann;             /* (N_max (N_max + 1) / 2) */
  const double* log_trans;             /* (2, 2 (width / 2) + 1, n_bins) */
  const double* freqs;                 /* (n_bins) */
  double* f0;                          /* out (B, F) */
  uint8_t* voiced_flag;                /* out (B, F) */
  double* voiced_prob;                 /* out (B, F) */
  void* ws; size_t ws_bytes;
} T2PyinArgs;
size_t t2_pyin_workspace_bytes(const T2PyinArgs* a);
int    t2_pyin(const T2PyinArgs* a, void* stream);
/* values (B, F) fp64 and durations (B, T_text) int64, both on the device -> out (B, T_text) fp32: for symbol j the mean
 * of the values[b, f] that are neither 0 nor NaN over f in [cum_j, cum_{j+1}) (cum = the row's running sum of
 * durations), summed in fp64 in frame order; 0 for a span without any.  Negative durations count as 0 and spans are cut
 * at F (the Python mirror refuses both).  One launch, no host synchronisation. */
int    t2_average_by_durations(const double* values, const int64_t* durations, int32_t B, int32_t F, int32_t T_text,
                               float* out, void* stream);

/* ---- Dynamic time warping (tacotron2_b200.dtw / mel_cepstral_distortion; DESIGN section 6.12) ---------------------
 * x (B, D, T_x) and y (B, D, T_y), both fp32 (dtype T2_DTW_F32) or both fp64 (T2_DTW_F64), row-major -> per row b the
 * cheapest monotonic path through C[i, j] = sqrt(sum_d (x[b, d, i] - y[b, d, j])^2) (fp64, summed in the order
 * d = 0 .. D - 1 without contraction) from (0, 0) to (L_x - 1, L_y - 1) with steps (1, 1), (0, 1), (1, 0) and unit
 * weights: D[0, 0] = C[0, 0], D[i, j] = C[i, j] + min(D[i-1, j-1], D[i, j-1], D[i-1, j]), ties to the diagonal, then
 * (i, j - 1), then (i - 1, j).  Row b reads only x[b, :, :L_x] and y[b, :, :L_y] (L = the lengths; a NULL array means
 * the full size; device lengths are clamped into [1, T], the Python mirror refuses them).
 * Out: cost (B) fp64 = D[L_x - 1, L_y - 1]; path (B, T_x + T_y - 1, 2) int64, the (i, j) pairs from (0, 0) on, padded
 * with -1; path_lengths (B) int64.  D > T2_DTW_MAX_DIM or T_x, T_y > T2_DTW_MAX_FRAMES are T2_ERR_UNSUPPORTED, other
 * bad sizes or a NULL pointer T2_ERR_INVALID, too small a workspace T2_ERR_WORKSPACE, before anything is launched.
 * 1 launch, no handle, no allocation, no host synchronisation.  Workspace: t2_dtw_workspace_bytes (0 for sizes the
 * call refuses): the 2-bit predecessor map, (T_x + T_y - 1) W 8 bytes per row with W = min(ceil(T_x / 32),
 * ceil(min(T_x, T_y) / 32) + 1), when it exceeds 96 KB (it stays in shared memory otherwise).
 * t2_mel_cepstra: mel (B, n_mel, T) fp32 / fp64 -> cep (B, n_cep, T) fp64, cep[b, k, t] = sum_m table[k, m] mel[b, m, t]
 * in the order m = 0 .. n_mel - 1 without contraction, for t < lengths[b] (NULL: T), 0 after; table (n_cep, n_mel) fp64
 * on the device, 1 <= n_cep < n_mel <= T2_DTW_MAX_DIM, T <= T2_DTW_MAX_FRAMES, B <= 65535.  1 launch. */
#define T2_DTW_MAX_FRAMES 8192
#define T2_DTW_MAX_DIM    1024
#define T2_DTW_F32        0
#define T2_DTW_F64        1
typedef struct T2DtwArgs {
  const void* x;                       /* (B, D, T_x) */
  const void* y;                       /* (B, D, T_y) */
  const int32_t* x_lengths;            /* (B) device or NULL */
  const int32_t* y_lengths;            /* (B) device or NULL */
  int32_t B, D, T_x, T_y, dtype;
  double* cost;                        /* out (B) */
  int64_t* path;                       /* out (B, T_x + T_y - 1, 2) */
  int64_t* path_lengths;               /* out (B) */
  void* ws; size_t ws_bytes;
} T2DtwArgs;
size_t t2_dtw_workspace_bytes(int32_t B, int32_t D, int32_t T_x, int32_t T_y, int32_t dtype);
int    t2_dtw(const T2DtwArgs* a, void* stream);
int    t2_mel_cepstra(const void* mel, int32_t dtype, const int32_t* lengths, int32_t B, int32_t n_mel, int32_t T,
                      const double* table, int32_t n_cep, double* cep, void* stream);

/* ---- WaveGlow vocoder inference (waveglow/glow.py: WaveGlow.infer, glow.py:251-293) ---------------
 * A separate handle: mel spectrogram (B, 80, T_mel) -> audio (B, 256 * T_mel).  Supported configurations (the published
 * one, waveglow/config.json, is the comment beside each field): n_mel_channels 80, n_group 8, wn_kernel_size 3,
 * wn_n_channels 128, 256, 384 or 512, wn_n_layers 1 ... 10, n_flows 1 ... 16, n_early_every >= 1 and n_early_size even,
 * leaving the last flow at least 2 channels.  t2_waveglow_create returns T2_ERR_UNSUPPORTED for anything else, before
 * any launch.
 * Precision tier: fp16 = 0 uses split-fp16 (hi + lo) operands with fp32 accumulation and fp32 state ("fp32 grade");
 * fp16 = 1 (a module converted with .half()) uses single fp16 operands with fp32 accumulation. */
typedef struct T2WaveGlow T2WaveGlow;   /* opaque: configuration + packed device-side weights */
typedef struct T2WaveGlowConfig {
  int32_t n_mel_channels;              /* 80  */
  int32_t n_flows;                     /* 12  */
  int32_t n_group;                     /* 8   */
  int32_t n_early_every;               /* 4   */
  int32_t n_early_size;                /* 2   */
  int32_t wn_n_layers;                 /* 8   */
  int32_t wn_kernel_size;              /* 3   */
  int32_t wn_n_channels;               /* 256 */
  int32_t fp16;                        /* 1: the weight table holds __half tensors (except convinv, always fp32) */
} T2WaveGlowConfig;

/* Entries of the WaveGlow weight table: the reference state_dict in its own order.  Weight-normed convolutions
 * contribute (bias, weight_g, weight_v); the library folds g * v / ||v|| when it packs.  After remove_weightnorm a
 * weight_g entry may be NULL and the weight_v entry is then the plain weight.  T2_WAVEGLOW_NUM_WEIGHTS is the published
 * configuration's count; t2_waveglow_num_weights gives any supported configuration's, 2 + n_flows (6 wn_n_layers + 9),
 * and 0 for a NULL or unsupported one. */
#define T2_WAVEGLOW_NUM_WEIGHTS 686
int32_t t2_waveglow_num_weights(const T2WaveGlowConfig* cfg);

int t2_waveglow_create(T2WaveGlow** out, const T2WaveGlowConfig* cfg, const void* const* weights, int32_t n_weights,
                       void* stream);
int t2_waveglow_refresh(T2WaveGlow* h, const void* const* weights, int32_t n_weights, void* stream);
int t2_waveglow_destroy(T2WaveGlow* h);

/* mel (B, 80, T_mel), fp32 or (io_half) __half.  lengths (B) int32 in mel frames or NULL: row b's samples
 * [0, 256 lengths[b]) equal an infer of that row's first lengths[b] frames alone; later samples are zero.
 * z (B, 8, 32 T_mel) fp32 or NULL: the standard-normal draws, channels in draw order (the last flow's channels, then
 * the early blocks from the last early flow down; published: 4, then flows 8 and 4); NULL => in-kernel Philox4x32-10 keyed by (seed, row, channel, group column).
 * row_seeds (B) device or NULL: row b's noise is keyed by (row_seeds[b], row 0, channel, group column) instead, the
 * draws of a B = 1 call with seed = row_seeds[b]; with z given it is T2_ERR_INVALID.
 * audio (B, 256 T_mel) out, in the mel's dtype. */
typedef struct T2WaveGlowArgs {
  const void* mel; int32_t B, T_mel; const int32_t* lengths; int32_t io_half;
  float sigma; const float* z; uint64_t seed;
  void* audio;
  void* ws; size_t ws_bytes;
  const uint64_t* row_seeds;
} T2WaveGlowArgs;
size_t t2_waveglow_workspace_bytes(const T2WaveGlow* h, int32_t B, int32_t T_mel);
int    t2_waveglow_infer(T2WaveGlow* h, const T2WaveGlowArgs* a, void* stream);

/* Windowed inference: the audio of some frames of a longer sequence from a window of its mel, bit-identical to the
 * same samples of t2_waveglow_infer over the whole sequence.  wg.mel holds frames [frame0, frame0 + T_mel) of the
 * sequence and wg.lengths are relative to the window (frames >= lengths[b] count as zero).  The audio of the
 * window-relative frames [out0, out1) is written to wg.audio, (B, 256 (out1 - out0)).  The noise is keyed by the
 * absolute group column 32 frame0 + t: Philox as above, or an injected wg.z (B, 8, 32 z_frames) read at absolute
 * columns, z_frames >= frame0 + T_mel.  at_end: the window ends where the sequence ends.
 * The audio of a frame depends on the halo_left frames before it and the halo_right after it: halo_right = ceil(n_flows
 * (2^wn_n_layers - 1) / 32), halo_left = halo_right + 3 (t2_waveglow_window_halo_config; 99 and 96 for the published
 * configuration, which t2_waveglow_window_halo returns).  The call returns T2_ERR_INVALID, launching nothing, when out0 is closer than the left
 * halo to a window start that is not the sequence's start (frame0 > 0), or out1 closer than the right halo to a
 * window end that is not the sequence's end (at_end = 0).  Workspace: t2_waveglow_workspace_bytes(h, B, T_mel).
 * t2_waveglow_infer is this call with frame0 = 0, [out0, out1) = [0, T_mel), z_frames = T_mel and at_end = 1. */
typedef struct T2WaveGlowWindowArgs {
  T2WaveGlowArgs wg;
  int32_t frame0;
  int32_t out0, out1;
  int32_t z_frames;
  int32_t at_end;
} T2WaveGlowWindowArgs;
void   t2_waveglow_window_halo(int32_t* left, int32_t* right);
/* The halos of the configuration `cfg` (fp16 is not read); T2_ERR_UNSUPPORTED, writing nothing, for an unsupported one. */
int    t2_waveglow_window_halo_config(const T2WaveGlowConfig* cfg, int32_t* left, int32_t* right);
int    t2_waveglow_infer_window(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, void* stream);

/* ---- HiFi-GAN generator inference (the V1 / V2 / V3 generators of jik876/hifi-gan, models.py) ---------------------
 * A separate handle: mel spectrogram (B, 80, T_mel) -> audio (B, 256 * T_mel).  Supported configurations (V1 is the
 * comment beside each field): 80 mels; 1 ... 8 upsampling stages with even rates whose product is 256 and kernels
 * k_i = 2 u_i; upsample_initial_channel and every stage's channel count (initial >> (i + 1)) multiples of 8 in
 * 8 ... 512; 1 ... 8 resblock kernels, each odd and at most 15, with 3 dilations (resblock 1) or 2 (resblock 2) whose
 * padding (k - 1) d / 2 is at most T2_HIFIGAN_MAX_PAD rows.  t2_hifigan_create returns T2_ERR_UNSUPPORTED for anything
 * else, before any launch.  Precision tier as WaveGlow's: fp16 = 0 split-fp16 operands ("fp32 grade"), fp16 = 1 (a
 * module converted with .half()) single fp16 operands; both accumulate in fp32. */
#define T2_HIFIGAN_MAX_STAGES 8
#define T2_HIFIGAN_MAX_KERNELS 8
#define T2_HIFIGAN_MAX_PAD 64
typedef struct T2HiFiGAN T2HiFiGAN;     /* opaque: configuration + packed device-side weights */
typedef struct T2HiFiGANConfig {
  int32_t n_mel_channels;                                       /* 80 */
  int32_t resblock;                                             /* 1 (ResBlock1) or 2 (ResBlock2) */
  int32_t n_upsamples;                                          /* 4 */
  int32_t upsample_rates[T2_HIFIGAN_MAX_STAGES];                /* 8, 8, 2, 2 */
  int32_t upsample_kernel_sizes[T2_HIFIGAN_MAX_STAGES];         /* 16, 16, 4, 4 */
  int32_t upsample_initial_channel;                             /* 512 */
  int32_t n_kernels;                                            /* 3 */
  int32_t resblock_kernel_sizes[T2_HIFIGAN_MAX_KERNELS];        /* 3, 7, 11 */
  int32_t resblock_dilation_sizes[T2_HIFIGAN_MAX_KERNELS][3];   /* (1, 3, 5) x 3; resblock 2 reads the first two */
  int32_t fp16;                                                 /* 1: the weight table holds __half tensors */
} T2HiFiGANConfig;

/* Entries of the weight table: the generator's state_dict in its own order, (bias, weight_g, weight_v) for every
 * convolution: conv_pre, ups.*, resblocks.* (ResBlock1: convs1.*, then convs2.*), conv_post.  A NULL weight_g entry
 * means the weight norm was removed and the weight_v entry is the plain weight.  weight_g is folded along dim 0, the
 * output channel of a Conv1d and the input channel of a ConvTranspose1d.  0 for a NULL or unsupported configuration. */
int32_t t2_hifigan_num_weights(const T2HiFiGANConfig* cfg);
int t2_hifigan_create(T2HiFiGAN** out, const T2HiFiGANConfig* cfg, const void* const* weights, int32_t n_weights,
                      void* stream);
int t2_hifigan_refresh(T2HiFiGAN* h, const void* const* weights, int32_t n_weights, void* stream);
int t2_hifigan_destroy(T2HiFiGAN* h);

/* mel (B, 80, T_mel), fp32 or (io_half) __half.  lengths (B) int32 in mel frames or NULL (values are clamped to
 * [0, T_mel]): row b's samples [0, 256 lengths[b]) equal a call on that row's first lengths[b] frames alone, bit for
 * bit; later samples are zero.  audio (B, 256 T_mel) out, in the mel's dtype.  B * (256 T_mel + the configuration's
 * guard rows) must stay below 2^30, else T2_ERR_INVALID.  Workspace: t2_hifigan_workspace_bytes(h, B, T_mel); nothing
 * is allocated and nothing waits for the device. */
typedef struct T2HiFiGANArgs {
  const void* mel; int32_t B, T_mel; const int32_t* lengths; int32_t io_half;
  void* audio;
  void* ws; size_t ws_bytes;
} T2HiFiGANArgs;
size_t t2_hifigan_workspace_bytes(const T2HiFiGAN* h, int32_t B, int32_t T_mel);
int    t2_hifigan_infer(T2HiFiGAN* h, const T2HiFiGANArgs* a, void* stream);

/* ---- WaveGlow denoiser (waveglow/denoiser.py: Denoiser, over stft.py:69-136 and audio_processing.py:7-56) -------
 * A separate handle holding the packed STFT bases.  The kernels are built for the reference default: filter_length
 * 1024, hop 256, win_length 1024, periodic Hann window; t2_denoiser_create returns T2_ERR_UNSUPPORTED for anything
 * else.  forward_basis and inverse_basis are the reference's windowed bases, fp32 (1026, 1, 1024) on the device.
 * Arithmetic: split-fp16 operands with fp32 accumulation (fp32 grade); the reference denoises in fp32. */
typedef struct T2Denoiser T2Denoiser;   /* opaque: packed device-side bases */
#define T2_WINDOW_HANN 0
typedef struct T2DenoiserConfig {
  int32_t filter_length;               /* 1024 */
  int32_t hop_length;                  /* 256  */
  int32_t win_length;                  /* 1024 */
  int32_t window;                      /* T2_WINDOW_HANN */
} T2DenoiserConfig;
int t2_denoiser_create(T2Denoiser** out, const T2DenoiserConfig* cfg, const float* forward_basis,
                       const float* inverse_basis, void* stream);
int t2_denoiser_refresh(T2Denoiser* h, const float* forward_basis, const float* inverse_basis, void* stream);
int t2_denoiser_destroy(T2Denoiser* h);
/* bias_spec (denoiser.py:36-38): bias_out (513) = the STFT magnitude of frame 0 of audio (n > 512 fp32 samples on the
 * device, reflect-padded by 512). */
int t2_denoiser_bias(T2Denoiser* h, const float* audio, int32_t n, float* bias_out, void* stream);

/* Denoiser.forward (denoiser.py:40-45): audio (B, n), fp32 or (io_half) __half -> out (B, 256 floor(n / 256)) fp32:
 * magnitudes lose strength * bias (513 fp32), clamped at 0, with the phase kept.  lengths (B) int32 in samples or NULL:
 * row b is denoised as its first lengths[b] samples alone (reflect-padded at its own end), and its output from sample
 * 256 floor(lengths[b] / 256) on is zero; a row of <= 512 samples cannot be padded and gives zeros.  Without lengths
 * n must exceed 512.  Amplitude: the GEMM operands are split fp16 values, so every sample must stay below 65504 in
 * magnitude (int16-scale audio up to 32767 is fine; any fp16 input is) and strength must be >= 0; larger values give
 * inf or NaN.  out must be 16-byte aligned (T2_ERR_INVALID otherwise).  Workspace: t2_denoiser_workspace_bytes(h, B, n). */
typedef struct T2DenoiserArgs {
  const void* audio; int32_t B, n; const int32_t* lengths; int32_t io_half;
  const float* bias; float strength;
  float* out;
  void* ws; size_t ws_bytes;
} T2DenoiserArgs;
size_t t2_denoiser_workspace_bytes(const T2Denoiser* h, int32_t B, int32_t n);
int    t2_denoiser_run(T2Denoiser* h, const T2DenoiserArgs* a, void* stream);

/* Windowed denoising: some output blocks of a longer sequence from a window of its audio, bit-identical to the same
 * samples of t2_denoiser_run over the whole sequence.  dn.audio holds samples [s0, s0 + n) of the sequence, s0 a
 * multiple of 256.  The output blocks [out0, out1), relative to the window (block k = samples 256 k ... 256 k + 255),
 * are written to dn.out, (B, 256 (out1 - out0)).  dn.lengths are relative to the window: lengths[b] in [0, n] ends
 * row b there; a negative or larger value (or NULL) ends it at the window's end when at_end, else the row goes on past
 * the window.  An output block depends on the 3 blocks of audio before it and the 3 after it
 * (t2_denoiser_window_halo: left, right).  The call returns T2_ERR_INVALID, launching nothing, when out0 is closer
 * than the left halo to a window start that is not the sequence's start (s0 > 0), or out1 closer than the right halo
 * to a window end that is not the sequence's end (at_end = 0).  Workspace: t2_denoiser_workspace_bytes(h, B, n).
 * t2_denoiser_run is this call with s0 = 0, [out0, out1) = [0, n / 256) and at_end = 1. */
typedef struct T2DenoiserWindowArgs {
  T2DenoiserArgs dn;
  int32_t s0;
  int32_t out0, out1;
  int32_t at_end;
} T2DenoiserWindowArgs;
void   t2_denoiser_window_halo(int32_t* left, int32_t* right);
int    t2_denoiser_run_window(T2Denoiser* h, const T2DenoiserWindowArgs* a, void* stream);

/* ---- STFT transform / inverse and Griffin-Lim (stft.py:69-141, audio_processing.py:59-75) -------------------------
 * They run on the T2Denoiser handle: it holds the packed STFT bases, so the same configuration rules apply (filter_length
 * 1024, hop 256, win_length 1024, periodic Hann; other configurations are refused by t2_denoiser_create with
 * T2_ERR_UNSUPPORTED) and the same arithmetic (split-fp16 operands, fp32 accumulation).  Each row's operands are scaled
 * by a power of two taken on the device from its largest magnitude (or sample) and the fp32 outputs undo it exactly:
 * inputs of any scale are supported away from fp32 overflow and underflow, and a power-of-two scale of a row's input
 * scales its output bit for bit.  Every row's output depends only on that row.  Invalid arguments return
 * T2_ERR_INVALID (too small a workspace T2_ERR_WORKSPACE) before anything is launched. */

/* transform (stft.py:69-94): audio (B, n) fp32 -> magnitude and phase (atan2), each (B, 513, n / 256 + 1) fp32.
 * lengths (B) int32 in samples or NULL: row b is transformed as its first lengths[b] samples alone (a value outside
 * [0, n] counts as n) and its frames from lengths[b] / 256 + 1 on are zero; a row of <= 512 samples cannot be
 * reflect-padded and gives zeros.  Without lengths n must exceed 512.
 * Workspace: t2_stft_transform_workspace_bytes(h, B, n). */
typedef struct T2StftTransformArgs {
  const float* audio; int32_t B, n; const int32_t* lengths;
  float* magnitude; float* phase;
  void* ws; size_t ws_bytes;
} T2StftTransformArgs;
size_t t2_stft_transform_workspace_bytes(const T2Denoiser* h, int32_t B, int32_t n);
int    t2_stft_transform(T2Denoiser* h, const T2StftTransformArgs* a, void* stream);

/* inverse (stft.py:96-136): magnitude and phase (B, 513, F) fp32, F >= 4 -> out (B, 256 (F - 1)) fp32, 16-byte
 * aligned.  lengths (B) int32 in frames or NULL: row b is the inverse of its first lengths[b] frames alone (a value
 * outside [0, F] counts as F), and its output from sample 256 (lengths[b] - 1) on is zero; a row of fewer than 4 frames
 * gives zeros.  Workspace: t2_stft_inverse_workspace_bytes(h, B, F). */
typedef struct T2StftInverseArgs {
  const float* magnitude; const float* phase; int32_t B, F; const int32_t* lengths;
  float* out;
  void* ws; size_t ws_bytes;
} T2StftInverseArgs;
size_t t2_stft_inverse_workspace_bytes(const T2Denoiser* h, int32_t B, int32_t F);
int    t2_stft_inverse(T2Denoiser* h, const T2StftInverseArgs* a, void* stream);

/* Griffin-Lim (audio_processing.py:59-75): signal = inverse(magnitude, inv.phase), then n_iters >= 0 times signal =
 * inverse(magnitude, phase of transform(signal)); out = the final signal.  inv.phase holds the initial angles; shapes
 * and lengths as t2_stft_inverse.  3 n_iters + 2 kernel launches, no host synchronisation.
 * Workspace: t2_griffin_lim_workspace_bytes(h, B, F). */
typedef struct T2GriffinLimArgs {
  T2StftInverseArgs inv;
  int32_t n_iters;
} T2GriffinLimArgs;
size_t t2_griffin_lim_workspace_bytes(const T2Denoiser* h, int32_t B, int32_t F);
int    t2_griffin_lim(T2Denoiser* h, const T2GriffinLimArgs* a, void* stream);

/* ---- self tests (libt2b200_selftest.so only: the same sources built with -DT2_SELFTEST; not part of the product
 * library) -------------------------------------------------------------------------------------------------
 * t2_selftest_event: the wgmma split-fp16 event engine's consumer plans and MMA chunk loop (event_mma, shared by the
 * persistent decoder's events and the decoder backward), on an event plan given as its consumers' row counts
 * (consumers_host[0..n_consumers), host memory; 1-3 consumers of 16 or 32 rows), run by the backward's skinny GEMM
 * kernel with one 64-row slice: C (64 x N) = A (64 x K) . W (N x K)^T fp32 with N the sum of the rows, W's
 * rows in consumer order, K a multiple of 64 up to 1024. */
#ifdef T2_SELFTEST
int t2_selftest_event(const float* A, const float* W, const int32_t* consumers_host, int32_t n_consumers, int32_t K,
                      float* C, void* stream);
/* Micro-benchmark: SM cycles for `reps` back-to-back wgmma of one warpgroup (M = 64, N in {32, 64, 128}, K = 16, fp16,
 * operands resident in shared memory) -> out_host[0] = issue cycles, out_host[1] = issue + completion cycles. */
int t2_selftest_mma_rate(int32_t M, int32_t N, int32_t reps, int32_t alternate_d, int64_t* out_host);
/* `reps` groups of `group` back-to-back MMAs, each group followed by a commit + a wait for it (one K chunk of a
 * streaming event): out_host[0] = total SM cycles. */
int t2_selftest_mma_group(int32_t M, int32_t N, int32_t group, int32_t reps, int64_t* out_host);
/* The training path's general tensor-core GEMM (gemm_tc.cu): row-major C = op(A) . op(B) + beta C, strided batch. */
int t2_selftest_gemm_tc(int32_t ta, int32_t tb, int32_t M, int32_t N, int32_t K, const float* A, int64_t lda,
                        const float* B, int64_t ldb, float* C, int64_t ldc, float beta, int32_t batch,
                        int64_t strideA, int64_t strideB, int64_t strideC, void* stream);
int t2_selftest_colsum(const float* X, int64_t ld, int64_t rows, int32_t cols, float* out, void* stream);
/* t2_waveglow_infer_window's own launch sequence for `a`, left after its first n_launches launches (0 ... 207: mel to
 * planes, the upsample GEMM, the initial tail, then per flow 11 ... 0 eight (gate GEMM, res/skip GEMM) pairs and a
 * tail), and the workspace as it then stands unpacked into fp32 device buffers; a NULL buffer is skipped.  Row
 * q = b * span + t, span = 32 T_mel + 128, rows = 128 ceil(B span / 128); channel c of the planes (spect, h, acts) is
 * hi + lo in the fp32-grade tier and hi in the fp16 tier.  skip and aud are not cleared between calls: rows no launch
 * has written yet hold what an earlier call left. */
int t2_selftest_waveglow_state(T2WaveGlow* h, const T2WaveGlowWindowArgs* a, int32_t n_launches, float* spect /* (rows, 640) */,
                               float* hbuf /* (rows, 256) */, float* acts /* (rows, 256) */, float* skip /* (rows, 256) */,
                               float* aud /* (rows, 8) */, void* stream);
#endif
/* ---- instrumentation ---------------------------------------------------------------------------------- */
/* After a T2_IMPL_PERSISTENT run with the same args / workspace: SM cycles spent per phase of the
 * persistent kernel, summed over steps, on three sample CTAs (out_host[3][24]; phase list in
 * decoder_persistent.cu); all zero after a run with limits, whose kernel keeps no profile.
 * Synchronises the device. */
int t2_decoder_profile(const T2DecoderArgs* a, int64_t* out_host);
/* number of kernels this library has launched since load (for bench.py's gpu_launches) */
int64_t t2_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* T2B200_H_ */
