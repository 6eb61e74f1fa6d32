/*
 * gigaam_b200 -- C ABI of the H100-native GigaAM hot path (libgigaam_b200.so).
 *
 * The reference (salute-developers/GigaAM) has no FFI of its own: the path is reached through Python
 * nn.Modules.  Each entry point below replaces the torch-op body of one of those modules; the Python
 * mirror classes in gigaam_b200/ (same names, constructor kwargs and state_dict keys as the
 * reference) bind them with ctypes.  See INTEGRATION.md for the reference-side binding.
 *
 *   gam_logmel        <- gigaam/preprocess.py:53-98   FeatureExtractor.forward (MelSpectrogram + log)
 *   gam_encode        <- gigaam/encoder.py:605-647    ConformerEncoder.forward (subsampling + N layers)
 *   gam_ctc_greedy    <- gigaam/decoder.py:18-21 + gigaam/decoding.py:56-96  CTCHead + CTCGreedyDecoding
 *   gam_rnnt_greedy   <- gigaam/decoder.py:41-47,85-102 + gigaam/decoding.py:128-207
 *   gam_ctc_log_probs <- gigaam/decoder.py:18-21      CTCHead.forward
 *   gam_rnnt_joint    <- gigaam/decoder.py:41-47      RNNTJoint.joint
 *   gam_rnnt_predict  <- gigaam/decoder.py:85-102     RNNTDecoder.predict (1-layer LSTM)
 *   gam_emo_head      <- gigaam/model.py:272-293      GigaAMEmo pooling + head + softmax
 *   gam_emo_frame_logits / gam_emo_spans              the same head over spans of a recording of any length
 *
 * Conventions: every pointer marked "device" is a CUDA device pointer on the handle's device; the
 * library never allocates or frees caller memory in the hot calls (the caller passes a workspace of
 * gam_workspace_bytes()); all work is enqueued on `stream` (a cudaStream_t passed as void*) and the
 * call returns without synchronising; int return, 0 = ok, negative = error (gam_last_error()).
 * A handle is bound to one device and is not thread-safe.  No CPU fallback exists.
 */
#ifndef GIGAAM_B200_H_
#define GIGAAM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gam_handle gam_handle;

typedef struct gam_config {
  /* preprocessor (gigaam/preprocess.py:60-65) */
  int32_t sample_rate, n_mels, n_fft, win_length, hop_length, center;
  /* encoder (gigaam/encoder.py:510-526) */
  int32_t feat_in, n_layers, d_model, n_heads, d_ff;
  int32_t subsampling;      /* 0 = conv2d, 1 = conv1d */
  int32_t subs_kernel_size; /* 3 (conv2d) */
  int32_t conv_kernel_size; /* depthwise taps: 31 or 5 */
  int32_t conv_norm;        /* 0 = batch_norm (folded into the depthwise conv), 1 = layer_norm */
  int32_t self_attention;   /* 0 = rotary, 1 = rel_pos (v1 checkpoints) */
  int32_t pos_emb_max_len;
  /* head (gigaam/decoder.py) */
  int32_t head;        /* 0 = none (ssl), 1 = ctc, 2 = rnnt, 3 = emo (pooled Linear head, gam_emo_head) */
  int32_t num_classes; /* V + 1, blank id = V; emo: the C classes, 1 <= C <= 256 */
  int32_t pred_hidden, joint_hidden, max_symbols;
  /* longest T' the handle encodes; 0 = GAM_REL_POS_MAX_T.  Larger values (up to pos_emb_max_len) need a rel_pos model's
   * pos_proj tables of 2*max_encoded_frames-1 rows */
  int32_t max_encoded_frames;
} gam_config;

/* One Conformer layer; all pointers device.  "h" = fp16 row-major [out, in]; "f" = fp32. */
typedef struct gam_layer_weights {
  const float *ln_ff1_g, *ln_ff1_b;
  const void* ff1_w1; /* h [d_ff, d] */
  const float* ff1_b1;
  const void* ff1_w2; /* h [d, d_ff] */
  const float* ff1_b2;
  const float *ln_att_g, *ln_att_b;
  const void* w_qk; /* h [2d, d] = [linear_q ; linear_k] */
  const float* b_qk;
  const void* w_v; /* h [d, d].  When w_v sits directly behind w_qk (one [3d, d] matrix) and b_v directly behind b_qk, the
                    * q, k and v projections run as a single launch */
  const float* b_v;
  const void* w_o; /* h [d, d] */
  const float* b_o;
  const float *ln_conv_g, *ln_conv_b;
  const void* pw1_w; /* h [2d, d], rows permuted so every 256-row tile is [128 value | 128 gate] */
  const float* pw1_b; /* f [2d], same permutation */
  const float* dw_w;  /* f [k, d]  depthwise taps, tap-major (eval BatchNorm folded in when conv_norm == 0) */
  const float* dw_b;  /* f [d] */
  const float *cn_g, *cn_b; /* conv LayerNorm affine (conv_norm == 1), else NULL */
  const void* pw2_w;  /* h [d, d] */
  const float* pw2_b;
  const float *ln_ff2_g, *ln_ff2_b;
  const void* ff2_w1;
  const float* ff2_b1;
  const void* ff2_w2;
  const float* ff2_b2;
  const float *ln_out_g, *ln_out_b;
  /* self_attention == 1 (rel_pos, gigaam/encoder.py:191-228) only, else NULL; w_qk / w_v are then unused */
  const void* w_qkv_rel;  /* h [4d, d] = [linear_q ; linear_q ; linear_k ; linear_v] */
  const float* b_qkv_rel; /* f [4d]    = [b_q + pos_bias_u ; b_q + pos_bias_v ; b_k ; b_v] */
  const void* pos_proj;   /* h [2*max-1, d]: linear_pos(pe(r)), row max-1-r for relative position r (pe =
                           * gigaam/encoder.py:318-326), max = gam_config.max_encoded_frames (0: GAM_REL_POS_MAX_T) */
} gam_layer_weights;

#define GAM_REL_POS_MAX_T 768 /* default longest T' (6 key blocks of 128 = 30.7 s of audio); see max_encoded_frames */
/* widest head d_k = d_model / n_heads each attention kernel runs (its per-warp Q and O fragments are specialised for
 * d_k / 16 k16 steps); gam_create refuses a wider one */
#define GAM_ROTARY_MAX_DK 48
#define GAM_REL_POS_MAX_DK 64
/* widest joint_hidden the fused RNN-T loss runs (gam_rnnt_loss*): its gradient kernels hold six 64-unit chunks of a hidden row
 * in registers, and at joint_hidden 344 with a 64-column strip the node kernel's dynamic shared memory is exactly the 227 KiB
 * per-block limit minus its row table */
#define GAM_RNNT_LOSS_MAX_JOINT_HIDDEN 344
/* widest pred_hidden gam_rnnt_predict_backward runs: its BPTT step keeps 5 pred_hidden floats of 4 utterances in the 48 KiB
 * of shared memory a launch gets by default (49 120 bytes at 614) */
#define GAM_PREDICT_BACKWARD_MAX_HIDDEN 614

typedef struct gam_weights {
  /* front end */
  const float* window;  /* f [n_fft]  (checkpoint buffer preprocessor.featurizer.0.spectrogram.window) */
  const float* dft_cos; /* f [n_fft/2+1, n_fft/2+1]  cos(2 pi k n / n_fft), row n, column k */
  const float* dft_sin; /* f [n_fft/2+1, n_fft/2+1]  sin(2 pi k n / n_fft) */
  const float* mel_fb;  /* f [n_fft/2+1, n_mels]     (checkpoint buffer ...mel_scale.fb) */
  /* subsampling (conv2d) */
  const float* sub1_w; /* f [C, 9]       encoder.pre_encode.conv.0.weight */
  const float* sub1_b; /* f [C] */
  const void* sub2_w;  /* h [C, 9*C]     conv.2.weight permuted to (out, kt, kf, in) */
  const float* sub2_b; /* f [C] */
  const void* sub_out_w; /* h [d, F2*C]  pre_encode.out.weight with K permuted from (c, f) to (f, c) */
  const float* sub_out_b;
  /* rotary tables f [pos_emb_max_len, d_k/2] */
  const float* rope_cos;
  const float* rope_sin;
  const gam_layer_weights* layers; /* HOST array of n_layers structs holding device pointers */
  /* CTC head, fp32 */
  const float* ctc_w; /* f [V+1, d] */
  const float* ctc_b;
  /* RNN-T head, fp32 */
  const float* rnnt_enc_w;     /* f [joint_hidden, d]   joint.enc.weight */
  const float* rnnt_enc_b;
  const float* rnnt_emb_gates; /* f [V+1, 4H]  embed(k) W_ih^T + b_ih + b_hh */
  const float* rnnt_whh_t;     /* f [H, 4H]    lstm.weight_hh_l0^T */
  const float* rnnt_wp_t;      /* f [H, joint_hidden]  joint.pred.weight^T */
  const float* rnnt_bp;
  const float* rnnt_wo;        /* f [V+1, joint_hidden] joint.joint_net.1.weight */
  const float* rnnt_bo;
  /* subsampling (conv1d, v3 checkpoints): weights permuted to (out, tap, in) */
  const void* c1d_w1;  /* h [d, k * feat_in]  encoder.pre_encode.conv.0.weight */
  const float* c1d_b1; /* f [d] */
  const void* c1d_w2;  /* h [d, k * d]        encoder.pre_encode.conv.2.weight */
  const float* c1d_b2; /* f [d] */
  /* tensor-core front end: split-precision DFT basis h [512, 3*Kp], Kp = n_fft rounded up to 64; every 256-row tile is
   * [128 cos rows | 128 sin rows] of bins tile*128.., K blocks [hi | hi | lo]; and the bin range of every mel filter */
  const void* dft_w;
  const int32_t* mel_lo; /* i32 [n_mels] first bin with a non-zero weight */
  const int32_t* mel_hi; /* i32 [n_mels] one past the last */
  /* emotion head (head == 3), fp32: Linear(d_model, C) applied to the mean of the encoder frames */
  const float* emo_w; /* f [C, d]  head.weight */
  const float* emo_b; /* f [C]     head.bias */
} gam_weights;

int gam_create(const gam_config* cfg, const gam_weights* w, int device, gam_handle** out);
void gam_destroy(gam_handle* h);
const char* gam_last_error(const gam_handle* h);
int gam_version(void);

/* frames of log-mel for n_samples (gigaam/preprocess.py:78-92) and encoder frames for M mel frames
 * (gigaam/encoder.py:77-90) -- host arithmetic */
int64_t gam_logmel_frames(const gam_handle* h, int64_t n_samples);
int64_t gam_encoded_frames(const gam_handle* h, int64_t mel_frames);

/* bytes of scratch gam_encode / gam_*_greedy need for a batch of B utterances of M mel frames */
int64_t gam_workspace_bytes(const gam_handle* h, int32_t B, int64_t mel_frames);

/* bytes of scratch gam_ctc_greedy / gam_rnnt_greedy need on their own (B utterances of T encoder frames) */
int64_t gam_decode_workspace_bytes(const gam_handle* h, int32_t B, int32_t T);
/* ... and the scored twins gam_ctc_greedy_scored / gam_rnnt_greedy_scored (>= gam_decode_workspace_bytes) */
int64_t gam_decode_scored_workspace_bytes(const gam_handle* h, int32_t B, int32_t T);

/* wav: device f32 [B, n_samples]  ->  mel: device f32 [B, n_mels, M] */
int gam_logmel(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, float* mel, void* stream);

/* Same result as gam_logmel on the tensor cores: frames -> fp16 (hi, lo) split -> one K-concatenated wgmma GEMM
 * against the split DFT basis with a |X|^2 epilogue -> sparse mel projection + log.  Needs scratch
 * (gam_logmel_workspace_bytes); gam_logmel (one fused CUDA-core kernel) needs none. */
int64_t gam_logmel_workspace_bytes(const gam_handle* h, int32_t B, int64_t n_samples);
int gam_logmel_tc(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, float* mel, void* workspace,
                  int64_t workspace_bytes, void* stream);

/* Varlen execution: lengths stay on the device (no host synchronisation, same launch sequence for every mix of lengths, so a
 * captured CUDA graph of the call is valid for all of them).  From the second subsampling stage on only the frames that
 * exist are computed (rows of the utterances packed back to back, cu_seqlens built by the first kernel of the call -- the
 * contract of apply_masked_flash_attn, gigaam/utils.py:103-155, applied to the whole Conformer block); frames t >= enc_len[b]
 * of `enc` are written as zeros.  A batch of ONE keeps its padded frames, like the reference (no attention mask for B == 1).
 * mel: device f32 [B, feat_in, M]; mel_len: device i64 [B]
 * -> enc: device f32 [B, T', d_model] (row-major; the reference's [B, d, T'] is its transpose(1,2) view)
 *    enc_len: device i32 [B].  n_layers_run < 0 runs the full stack; 0..n_layers stops early (tests). */
int gam_encode(gam_handle* h, const float* mel, const int64_t* mel_len, int32_t B, int64_t M, void* workspace,
               int64_t workspace_bytes, float* enc, int32_t* enc_len, int32_t n_layers_run, void* stream);

/* enc: device f32 [B, T, d_model]; enc_len: device i32 [B]
 * -> ids / frames: device i32 [B, max_out], counts: device i32 [B] */
int gam_ctc_greedy(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                   int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                   void* stream);
int gam_rnnt_greedy(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                    int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                    void* stream);

/* Scored greedy decoding: the same ids / frames / counts as gam_*_greedy, bit for bit, plus how sure the model was.
 * A decision row is one logit row the greedy rule evaluates: CTC, every frame t < enc_len[b]; RNN-T, every joint row of
 * the loop of gigaam/decoding.py:184-205, emissions and blanks alike (a frame that reaches max_symbols emissions has no
 * closing blank row).  l(row) = log_softmax(row)[label] for the label the greedy rule picks = -log sum_c exp(z_c - z_max)
 * on a finite row; NaN on a row with a NaN or +inf logit or with only -inf logits (the label stays 0).
 *   token_logp device f32 [B, max_out]: l of the row that emitted token i (CTC: the first frame of the token's run).
 *   path_logp  device f32 [B]: sum of l over all decision rows of utterance b (fp64 accumulation; NaN if any row was).
 *   path_rows  device i32 [B]: the number of those rows.
 * An utterance's scores are bit-identical whatever batch it is decoded in.  Stream-ordered, no host sync, capturable in a
 * CUDA graph; workspace: gam_decode_scored_workspace_bytes. */
int gam_ctc_greedy_scored(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                          int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                          float* token_logp, float* path_logp, int32_t* path_rows, void* stream);
int gam_rnnt_greedy_scored(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                           int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                           float* token_logp, float* path_logp, int32_t* path_rows, void* stream);

/* Resumable greedy decoding: decode an utterance in consecutive chunks of frames, with the decoder's state carried in device
 * memory between calls, so that a recording of any length is decoded as one utterance while only a chunk of encoder output
 * is alive (GigaAMASR.transcribe_windowed).
 *
 * A decoding stream's state is one record of gam_decode_state_bytes(h) bytes: everything the greedy loop keeps across a
 * frame boundary.  RNN-T: h, c, W_p h + b_p, the last label, whether that label's LSTM step is still pending (a frame that
 * ended on its max_symbols-th emission), the token count and, when scored, the fp64 path sum and row count.  CTC: the
 * previous frame's label (a repeat across a chunk edge collapses), the token count, the fp64 partial path sums and the row
 * count.  gam_decode_state_init writes n fresh records (a new utterance) back to back at `state`.
 *
 * One call: row b decodes local frames [lo[b], hi[b]) (clamped to [0, T]) of enc[b] (device f32 [B, T, d_model], gam_encode's
 * layout), continuing stream b from state + b * gam_decode_state_bytes(h) and leaving the updated record there.  lo, hi and
 * frame_base are device i32 [B].
 *   ids / frames  device i32 [B, max_out]: tokens are appended at counts[b] (device i32 [B], read and written); frames are
 *                 frame_base[b] + t.  Tokens past max_out are dropped, counts[b] stops at max_out and the record keeps the
 *                 true count, so an overflow can be detected.
 *   token_logp    device f32 [B, max_out], or NULL for the unscored decoder, which writes none of the outputs below.
 *   path_logp / path_rows  device f32 / i32 [B]: the stream's running totals (gam_*_greedy_scored's definitions).
 *   frame_logp / frame_rows  device f64 / i32 [B, frame_pitch]: at frame_base[b] + t, the sum of l over the decision rows of
 *                 that frame and their number (CTC: one row per frame).
 * lo[b] == hi[b] leaves row b's record and outputs untouched.  Splitting [0, L) into consecutive ranges and decoding them in
 * order gives ids, frames, counts, token_logp, path_logp and path_rows bit-identical to one gam_*_greedy(_scored) call over
 * the same L frames, and frame_rows sums to path_rows.  Every row of enc is labelled / projected (the ranges live on the
 * device); workspace: gam_decode_resume_workspace_bytes.  Stream-ordered, no host sync, capturable in a CUDA graph. */
int64_t gam_decode_state_bytes(const gam_handle* h);
int gam_decode_state_init(gam_handle* h, void* state, int32_t n, void* stream);
int64_t gam_decode_resume_workspace_bytes(const gam_handle* h, int32_t B, int32_t T);
int gam_ctc_greedy_resume(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                          const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                          int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                          double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, void* stream);
int gam_rnnt_greedy_resume(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                           const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                           int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                           double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, void* stream);

/* Phrase boosting for RNN-T greedy decoding: gam_rnnt_greedy_resume steered by a boost graph (GigaAMASR.transcribe(boost=)).
 *
 * A boost graph is a dense automaton over the vocabulary: S states (1 <= S <= 65 536), boost_next device i32 [S, V1] and
 * boost_bonus device f32 [S, V1] (V1 = V + 1 columns, blank included); state 0 is the initial state.  Stream b is in one
 * state q, kept in its decoding record (bytes the RNN-T decoder does not otherwise use; gam_decode_state_init's zeros are
 * state 0, so the record keeps its size).
 *   - At every decision row in state q the label is the greedy rule (first maximal index; label 0 on a row with a NaN or +inf
 *     value or only -inf values) applied to fp32(z_v + bonus[q, v]) instead of z_v.  The blank column is ignored: blank gets
 *     no bonus, and emitting blank does not change q.
 *   - On emitting token v, q becomes boost_next[q, v]; an entry outside [0, S) sends the stream to state 0.
 *   - Scores stay the model's own: token_logp, path_logp / path_rows and frame_logp / frame_rows are log_softmax(z)[label] of
 *     the unboosted row (NaN by the unboosted rule where the label is 0 by the non-finite rule).  With finite bonuses a row with
 *     a non-finite logit decides as it does without boosting.
 *   - With every bonus 0, every output and the record outside q are bit-identical to gam_rnnt_greedy_resume's.
 * Arguments, scoring (token_logp non-NULL), workspace and the chunking rule are gam_rnnt_greedy_resume's; q is carried across
 * chunks in the record.  Refused: a model without an RNN-T head, NULL tables, S outside [1, 65 536], and everything the resume
 * call refuses.  The tables take S * V1 * 8 bytes; each CTA keeps its class slice of bonus[q] per utterance in shared memory. */
int gam_rnnt_greedy_boost(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                          const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                          int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                          double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, const int32_t* boost_next,
                          const float* boost_bonus, int32_t n_states, void* stream);

/* ---- the heads' forward passes, for callers that run their own search (LM beam search, N-best rescoring, forced
 * alignment, lattice scoring).  fp32 CUDA-core arithmetic like the reference's heads; no workspace except for the joint.
 *
 * CTC posteriors: enc: device f32 [B, T, d_model] (gam_encode's layout)
 *   -> log_probs: device f32 [B, T, V+1] = log_softmax(W enc + b) over the last axis.  Every frame is computed; frames at or
 *   past enc_len hold zeros in gam_encode's output and so give log_softmax(b).
 * Non-finite logits follow torch.log_softmax, here and in gam_rnnt_joint / gam_rnnt_align_scores: a -inf logit (e.g. a -inf
 * bias, which bans a class) gives -inf at its class and finite log-probs elsewhere; a row with a NaN or +inf logit, or with
 * every logit -inf, is all NaN. */
int gam_ctc_log_probs(gam_handle* h, const float* enc, int32_t B, int32_t T, float* log_probs, void* stream);

/* RNN-T joint lattice: enc: device f32 [B, T, d_model]; dec: device f32 [B, U, pred_hidden] (prediction-network outputs)
 *   -> out: device f32 [B, T, U, V+1] = log_softmax(W_o relu(W_e enc[b,t] + b_e + W_p dec[b,u] + b_p) + b_o).
 * workspace: device scratch of at least gam_rnnt_joint_workspace_bytes(B, T, U) bytes (the two projections); the
 * [B, T, U, joint_hidden] hidden tensor is never stored.  Offsets are 64-bit: out may exceed 2^31 elements.
 * Needs joint_hidden % 4 == 0 and <= 736 (the hidden tile lives in shared memory), pred_hidden % 16 == 0.  Non-finite
 * logits as gam_ctc_log_probs: -inf only at a -inf logit's class, all NaN for a row with a NaN or +inf logit (relu keeps
 * a NaN of enc or dec, so it reaches every row that reads it).
 * gam_rnnt_joint_workspace_bytes returns -1 for a handle without an RNN-T head or non-positive sizes. */
int64_t gam_rnnt_joint_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_joint(gam_handle* h, const float* enc, const float* dec, int32_t B, int32_t T, int32_t U, void* workspace,
                   int64_t workspace_bytes, float* out, void* stream);

/* RNN-T prediction network, U sequential LSTM steps (gate order i, f, g, o):
 *   x: device i64 [B, U] label ids, or NULL = one step (U must be 1) from the all-zero embedding;
 *   h0, c0: device f32 [B, pred_hidden] each, or NULL = zeros;
 *   -> g: device f32 [B, U, pred_hidden] (hidden state after every step), h1, c1: device f32 [B, pred_hidden] (final state).
 * An utterance with an id outside [0, V] gets NaN in all of its g, h1 and c1; the others are unaffected and the call
 * succeeds.  One launch per step. */
int gam_rnnt_predict(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, float* g, float* h1,
                     float* c1, void* stream);
/* gam_rnnt_predict (same bits) that also keeps the cell state of every step: c_seq device f32 [U, B, pred_hidden], the
 * operand gam_rnnt_predict_backward needs. */
int gam_rnnt_predict_train(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, float* g,
                           float* h1, float* c1, float* c_seq, void* stream);

/* ---- alignment of known transcripts: where in the audio a given token sequence lies, and how well the audio supports it.
 * Notation: T_b = enc_len[b] and U_b = target_len[b], each clamped to [0, T] / [0, U]; y_1..y_U_b are utterance b's target ids,
 * each in [0, V); blank = V (V + 1 = num_classes).  Every score is fp32 and comes from the caller.
 *
 * CTC (gam_ctc_align): states l' = (blank, y_1, blank, ..., y_U_b, blank), S = 2 U_b + 1.  State s is entered from s and s - 1,
 * and from s - 2 when l'_s != blank and l'_s != l'_{s-2}.  Paths start in state 0 or 1 at t = 0 and end in S - 1 or S - 2 at
 * t = T_b - 1.  Viterbi: v(0, s) = lp[0, l'_s] for s < 2, -inf elsewhere; v(t, s) = lp[t, l'_s] + max over the predecessors,
 * the max taken in the order s, s - 1, s - 2 with a later candidate replacing the current one only when strictly greater (on
 * ties, staying wins), then one fp32 add.  The final state is S - 1 unless v(T_b - 1, S - 2) > v(T_b - 1, S - 1) strictly.
 * Forward: the same recursion with log-sum-exp (-inf, never NaN, for all -inf operands); log_likelihood = logsumexp of the
 * final states = -F.ctc_loss(..., reduction="none").
 *
 * RNN-T (gam_rnnt_align): nodes (t, u), t < T_b, u <= U_b; blank(t, u) = log_softmax(joint(t, u))[V] and label(t, u) =
 * log_softmax(joint(t, u))[y_{u+1}], u < U_b, with joint(t, u) the row gam_rnnt_joint computes for dec = predict(cat[blank, y]).
 * Viterbi: v(0, 0) = 0, v(t, u) = max(v(t-1, u) + blank(t-1, u), v(t, u-1) + label(t, u-1)), one fp32 add per candidate, the
 * blank edge winning ties; no max_symbols cap.  viterbi_logp = v(T_b - 1, U_b) + blank(T_b - 1, U_b).  Forward: the same with
 * log-sum-exp; log_likelihood = -torchaudio rnnt_loss(..., reduction="none") on the log-prob lattice.
 *
 * Outputs per utterance b (frames / token_logp have row pitch U; entries i >= U_b are -1 / -inf):
 *   frames [B, U] i32: CTC, the first frame of token i's run on the Viterbi path; RNN-T, the frame at which token i is emitted
 *     (the greedy decoders' convention, so gam_group_words takes them with counts = target_len);
 *   token_logp [B, U] f32: CTC, lp at that frame; RNN-T, label(t, i) on the emitting edge;
 *   viterbi_logp [B], log_likelihood [B] f32; path_rows [B] i32: the edges on a path, T_b for CTC and T_b + U_b for RNN-T.
 * No path (CTC: T_b = 0 or T_b < U_b + adjacent repeats; RNN-T: T_b = 0), or a Viterbi score of -inf: both scores -inf, every
 * frame -1 and every token_logp -inf.  U_b = 0 is the all-blank path.  A NaN in any score the recursion reads (CTC: lp[t, blank]
 * and lp[t, y_i], t < T_b; RNN-T: blank(t, u) for t < T_b - 1, u <= U_b, label(t, u) for t < T_b, u < U_b, and
 * blank(T_b - 1, U_b)), or a CTC target id outside [0, V), makes both scores and every token_logp NaN and every frame -1;
 * entries that are not read never affect the result.  One CTA per utterance with fixed orders and no atomics: an utterance's
 * results are bit-identical in any batch and on every call.  Stream-ordered, no host synchronisation, capturable in a CUDA
 * graph.  Limits: U <= 4096 tokens, T <= the handle's max_encoded_frames; larger sizes are refused.  The workspaces hold the
 * backpointers (2 bits per CTC (t, s), 1 bit per RNN-T node); *_workspace_bytes return -1 for bad sizes or a handle without
 * the head.
 *
 * gam_ctc_align: log_probs [B, T, V+1] (gam_ctc_log_probs), enc_len [B], targets [B, U], target_len [B], all device. */
int64_t gam_ctc_align_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_ctc_align(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets, const int32_t* target_len,
                  int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                  float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream);
/* gam_ctc_align for recordings of any length: the same arguments, definitions, rules and outputs as gam_ctc_align, and on
 * every input gam_ctc_align accepts the same bits.  Only these differ:
 *   - limits: U <= 65536 tokens; T is bounded only by int32 and the workspace (not by max_encoded_frames);
 *   - one thread-block cluster of C <= 16 CTAs per utterance, C the smallest whose share of the 2U + 1 states (a multiple of
 *     16) fits in shared memory at 20 bytes per state; frame boundaries are exchanged through distributed shared memory;
 *   - workspace: B * T * ceil((2U + 1) / 16) * 4 bytes of backpointers (2.95 GB for T = 90 000, U = 65 536), rounded up to
 *     1 KiB; *_workspace_bytes returns -1 for bad sizes, U > 65536 or a handle without a CTC head.
 * Stream-ordered, no host synchronisation, capturable in a CUDA graph. */
int64_t gam_ctc_align_long_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_ctc_align_long(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets, const int32_t* target_len,
                       int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                       float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream);
/* gam_ctc_align_long for a text that only partly matches the recording: audio between lines that the text lacks is left
 * unaligned and reported.  An exact Viterbi (and forward) over the same states, transitions, tie rules and outputs as
 * gam_ctc_align_long; only what some blank states emit changes.
 *   - line_edges [B, U] u8 (device; may be NULL when U == 0): bit 0 = token i starts a line, bit 1 = it ends one.
 *   - Boundary states: state 0, state 2 U_b, the blank just before every token that starts a line and the blank just after
 *     every token that ends one.  (Between two charwise lines joined by a space token, those are the blanks on both sides of
 *     the space; the space itself is still required.)
 *   - Emission: at frame t a boundary state emits e_t = max(lp[t, blank], m[t] + log_theta) in both recursions, where
 *     m[t] = max_c lp[t, c] as gam_ctc_spot computes it (exact; a zero max is +0) and m[t] + log_theta is one fp32 add.  Every
 *     other state emits lp[t, l'_s] as before.
 *   - log_theta: the fp32 log of a threshold theta in (0, 1], a per-frame likelihood ratio to the greedy decoder as in
 *     gam_ctc_spot; -inf is accepted and gives gam_ctc_align_long's graph (on NaN-free input its bits, and no frame flagged).
 *     NaN and values > 0 are refused.
 *   - NaN rule: a recording reads the whole row lp[t, 0..V] of every frame t < T_b, so a NaN anywhere in those rows poisons it,
 *     with gam_ctc_align_long's outputs for a poisoned recording.
 * Outputs, besides gam_ctc_align_long's:
 *   unmatched [B, T] u8: 1 where the Viterbi path sits in a boundary state at frame t and m[t] + log_theta > lp[t, blank]
 *     strictly (a tie is matched), else 0; 0 at every t >= T_b and for a recording without a path or poisoned;
 *   unmatched_rows [B] i32: the number of unmatched frames;
 *   unmatched_logp [B] f32: the fp32 sum of m[t] + log_theta over the unmatched frames in frame order (0 when there are none,
 *     NaN for a poisoned recording).
 * Workspace: gam_ctc_align_long's backpointers plus B * T * 4 bytes of m[t], each rounded up to 1 KiB; *_workspace_bytes
 * returns -1 where gam_ctc_align_long_workspace_bytes does.  Two launches (the pre-pass that fills m, then the sweep), fixed
 * orders and no atomics: the same bits at every cluster size and in any batch.  Stream-ordered, no host synchronisation,
 * capturable in a CUDA graph.  Refuses everything gam_ctc_align_long refuses. */
int64_t gam_ctc_align_long_gaps_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_ctc_align_long_gaps(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                            const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                            void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp, float* viterbi_logp,
                            float* log_likelihood, int32_t* path_rows, uint8_t* unmatched, int32_t* unmatched_rows,
                            float* unmatched_logp, void* stream);
/* gam_ctc_align_long_gaps for a text that contains lines the recording lacks: a whole line may be skipped.  The graph is
 * gam_ctc_align_long_gaps' (the same states, transitions, emissions with the boundary states, tie rules, NaN rule and
 * outputs) with one more kind of edge:
 *   - Lines come from line_edges: a token with bit 1 set ends a line.  The exit state of the i-th such token j_i is the
 *     blank just after it, x_i = 2 (j_i + 1).  The skip source is e_i = x_{i-1}, or state 0 for the first line, and
 *     n_i = (x_i - e_i) / 2 is the number of tokens the edge jumps: the line and any joining token before it (such as the
 *     space between charwise lines).  Skips of consecutive lines chain, since x_i = e_{i+1}.
 *   - Edge: (t - 1, e_i) -> (t, x_i) with weight pen_i = fp32(n_i) * log_psi, one fp32 multiply.  x_i emits what it emits
 *     without the edge (the gap emission included).
 *   - Viterbi at x_i: the candidates are compared in the order stay, s - 1, skip, a later one winning only when strictly
 *     greater; the skip candidate is the fp32 add v(t - 1, e_i) + pen_i.  Forward: f(t, x_i) = e_t + lse3(f(t - 1, x_i),
 *     f(t - 1, x_i - 1), f(t - 1, e_i) + pen_i), operands in that order.
 *   - log_psi: the fp32 log of a threshold psi in (0, 1]; -inf is accepted and gives every output of
 *     gam_ctc_align_long_gaps bit for bit (on input without +inf scores).  NaN and values > 0 are refused.
 *   - The initial and final states are unchanged: skipping the first line costs one frame in state 0, and skipping the last
 *     line lands on 2 U_b.  A text may have a path with skips where it had none without.
 * Outputs, besides gam_ctc_align_long_gaps':
 *   tokens jumped by a skip edge on the Viterbi path have frame -1 and token_logp -inf;
 *   skipped_rows [B] i32: the number of skip edges on the path;
 *   skip_logp [B] f32: the fp32 sum of their pen_i in frame order (0 without a path, NaN for a poisoned recording).
 * Workspace: gam_ctc_align_long_gaps' (the sources are found again from line_edges); *_workspace_bytes returns what
 * gam_ctc_align_long_gaps_workspace_bytes returns.  The same launches, orders and guarantees as gam_ctc_align_long_gaps: the
 * same bits at every cluster size and in any batch, no host synchronisation, capturable in a CUDA graph.  Refuses a NaN or
 * positive log_psi, a NULL skipped_rows or skip_logp, and everything gam_ctc_align_long_gaps refuses. */
int64_t gam_ctc_align_long_skips_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_ctc_align_long_skips(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                             const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                             float log_psi, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                             float* viterbi_logp, float* log_likelihood, int32_t* path_rows, uint8_t* unmatched,
                             int32_t* unmatched_rows, float* unmatched_logp, int32_t* skipped_rows, float* skip_logp, void* stream);
/* ---- CTC keyword spotting: where in a recording each of K keywords was said, and how sure that is.  One exact Viterbi
 * per (recording, keyword) over the caller's fp32 log-probs; no hypothesis search.
 *
 * Recording b has lp[t, c] = log_probs[b, t, c], t < T_b = clamp(enc_len[b], 0, T); blank = V (V + 1 = num_classes).
 * Keyword k has tokens y_1..y_U, U = keyword_len[k], 1 <= U <= Umax <= 64, ids in [0, V) (keywords [k, i - 1] = y_i).
 *   States: y_1, blank, y_2, blank, ..., y_U, so S = 2U - 1; even s is token y_{s/2+1}, odd s the blank between two tokens,
 *     l_s its label.  There is no leading or trailing blank: a keyword starts on its first token and ends on its last.
 *   Transitions: state s is entered from s and from s - 1; an even s >= 2 also from s - 2 when y_{s/2+1} != y_{s/2} (a
 *     repeated token needs the blank between its two copies, so U = 1 and repeats have no skip).
 *   Cost: m[t] = max_c lp[t, c], exact (a zero max is +0); c(t, s) = lp[t, l_s] - m[t], one fp32 subtraction, <= 0, and 0 on
 *     the state whose label the greedy decoder picks at t.
 *   Recursion, fp32, one add per value, v(-1, s) = -inf:
 *     v(t, 0) = c(t, 0) + max(v(t-1, 0), 0): the path continues, or a fresh one starts at t (only when 0 > v(t-1, 0)
 *       strictly: on a tie the path continues, which keeps the earlier start);
 *     v(t, s > 0) = c(t, s) + the max over the predecessors, taken in the order s, s - 1, s - 2 with a later candidate
 *       replacing the current one only when strictly greater.
 *     Every state carries the start frame of its best path (the frame its fresh start was taken).
 *   NaN frames: a frame whose row lp[t, 0..V] holds a NaN is a barrier: v(t, s) = -inf for every s, so no path crosses it.
 *     (Infinite entries are not special: the arithmetic above applies as written.)
 *   End score: E(t) = v(t, S - 1), the best path that ends on y_U at t, with start frame a(t).  E(t) = log p(keyword path) -
 *     log p(best unconstrained path) over frames [a(t), t]; exp(E / U) is the per-token likelihood ratio to greedy, 1.0
 *     exactly where the greedy decoder writes the keyword.
 *   Detections: tau = fp32(U) * fp32(log threshold) (the log rounded once to fp32, computed on the host); frames t < T_b are
 *     scanned in order, and each with E(t) >= tau (so never a NaN or -inf one) is a candidate [a(t), t + 1) with score E(t).
 *     A candidate that overlaps the pending detection (a(t) < its end) replaces it only when its score is strictly greater,
 *     so ties keep the earlier end; a candidate that does not overlap emits the pending detection and becomes pending; the
 *     last pending detection is emitted after frame T_b - 1.  A greedy word thus spans [first frame of its first token's run,
 *     first frame of its last token's run + 1), the gam_group_words convention.
 *   T_b = 0, or a keyword longer than the frames that can hold it, gives no detection.
 * Outputs, per (b, k) at row (b K + k) of pitch max_det, in time order: det_start / det_end [B, K, max_det] i32 (frames,
 *   end exclusive), det_score [B, K, max_det] f32 (E), det_count [B, K] i32.  det_count is the true count even when it exceeds
 *   max_det; only the first max_det detections are stored, and entries past the stored ones are -1 / -1 / -inf.  A keyword
 *   with an id outside [0, V) or a length outside [1, Umax] gets count 0 and -1 / -1 / NaN in every entry; the call succeeds.
 * Refused (gam_last_error): a handle without a CTC head, B outside [1, 65535], T < 1, K < 1, Umax outside [1, 64], a
 *   threshold outside (0, 1] or NaN, max_det < 1, and a num_classes whose frame does not fit in shared memory.
 * All pointers are device memory; log_probs [B, T, V+1] (gam_ctc_log_probs, or stitched windows), enc_len [B], keywords
 * [K, Umax] i32, keyword_len [K] i32.  Fixed orders, no atomics: a (recording, keyword) pair's outputs are bit-identical
 * whatever else is in the batch and in whatever order the keywords come.  No workspace, no host synchronisation,
 * capturable in a CUDA graph.  T is bounded only by int32 (not by max_encoded_frames). */
int gam_ctc_spot(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                 const int32_t* keyword_len, int32_t K, int32_t Umax, float threshold, int32_t max_det, int32_t* det_start,
                 int32_t* det_end, float* det_score, int32_t* det_count, void* stream);
/* Resumable keyword spotting: gam_ctc_spot over a stream's frames in consecutive calls (live audio), with each (stream,
 * keyword) pair's search carried in device memory between them.  gam_ctc_spot itself is one such call from fresh records.
 *
 * A record is gam_ctc_spot_state_bytes(h, Umax) bytes: the pending detection (whether there is one, its start, end and
 * score), the true count of detections emitted so far, and every state's score v and start frame.
 * gam_ctc_spot_state_init writes n x K fresh records ([n, K, record], stream-major) at `state`.
 *
 * One call: row b walks local frames [lo[b], hi[b]) (clamped to [0, T]) of log_probs[b] ([B, T, V+1]) as stream frames
 * frame_base[b] + t, keyword k continuing from state + (b K + k) record_bytes and leaving the updated record there.  lo, hi,
 * frame_base and finish are device i32 [B].  Start and end frames, in records and outputs, are stream frames.
 *   det_*         as gam_ctc_spot's; detections emitted by the call are appended at det_count[b, k] (read and written), which
 *                 stops at max_det; the record keeps the true count.  Nothing else in det_* is written.
 *   pend_*        device i32 / i32 / f32 [B, K], or all three NULL: the pending detection after the call (start, end, score),
 *                 or -1 / -1 / -inf when there is none.  A pending detection may still be replaced by a better overlapping one.
 *   finish[b]     nonzero: the stream ends with this call, and its pending detection is emitted.  Without finish, the pending
 *                 detection is emitted early when no state with a finite score has a start frame before its end: no later
 *                 candidate can overlap it, so the detections and their order are exactly gam_ctc_spot's over the whole stream.
 * Splitting a stream's frames [0, L) into consecutive ranges, the last call with finish, gives gam_ctc_spot's detections over
 * the L frames bit for bit.  A keyword with a bad id or length gets no detections and a pending -1 / -1 / NaN.
 * Refused (gam_last_error): what gam_ctc_spot refuses, plus a NULL lo, hi, frame_base, finish or state, a record_bytes other
 * than gam_ctc_spot_state_bytes(h, Umax), and pend_* that are not all given or all NULL.  gam_ctc_spot_state_bytes returns -1
 * for a handle without a CTC head or a Umax outside [1, 64].  No workspace, no host synchronisation, capturable in a CUDA
 * graph. */
int64_t gam_ctc_spot_state_bytes(const gam_handle* h, int32_t Umax);
int gam_ctc_spot_state_init(gam_handle* h, void* state, int32_t n, int32_t K, int32_t Umax, void* stream);
int gam_ctc_spot_resume(gam_handle* h, const float* log_probs, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                        const int32_t* frame_base, const int32_t* finish, const int32_t* keywords, const int32_t* keyword_len, int32_t K,
                        int32_t Umax, float threshold, int32_t max_det, void* state, int64_t record_bytes, int32_t* det_start,
                        int32_t* det_end, float* det_score, int32_t* det_count, int32_t* pend_start, int32_t* pend_end,
                        float* pend_score, void* stream);
/* ---- CTC hotwords: the keywords gam_ctc_spot found replace the greedy words they outscore.  No hypothesis search: the greedy
 * output changes only where a stored detection beats it by the margin the threshold states.
 *
 * Recording b's inputs: lp, T_b, blank and the keywords y (U tokens, S = 2U - 1 states) as in gam_ctc_spot; the greedy tokens
 * (id_i, f_i), i < n = clamp(counts[b], 0, max_out), frames strictly increasing in [0, T); flag(id) = token_flags[id]
 * (gam_group_words' table: 1 the piece is " ", 2 it starts with U+2581; 0 for an id outside [0, V)); and every stored
 * detection (k, j < min(det_count[b, k], max_det)) of gam_ctc_spot at the same threshold: span [s, e), score E.
 *   1. Gain: G = E - tau in fp32, tau = fp32(U) * fp32(log threshold) (spot's tau), so G >= 0.
 *   2. Replaced range: [i0, i1) = the greedy tokens with f_i in [s, e) (binary searches over the frames); space tokens (flag 1)
 *      at either end are removed from the range and stay in the output.
 *   3. Eligible: i1 > i0 (nothing is inserted into silence) and i0 and i1 are word boundaries.  p is a word boundary when
 *      p = 0 or p = n, token p - 1 is a space, token p is a space, or token p starts a SentencePiece word (flag 2).  So a
 *      keyword is never spliced into part of a longer word.
 *   4. Selection: eligible candidates in the order G descending, then s ascending, then the longer keyword, then the
 *      lexicographically smaller ids, then the smaller k; each is accepted when [s, e) overlaps no accepted span.  Only exact
 *      duplicate keywords reach the last tie-break, and they splice the same tokens: the output does not depend on the
 *      keyword order or on the batch.
 *   5. Identity: an accepted candidate whose ids[i0, i1) already equal y keeps the greedy tokens, frames and scores bit for bit
 *      (it still blocks the candidates that overlap it).
 *   6. Splice: otherwise tokens [i0, i1) are replaced by y.  The traced path is the keyword's best path over [s, e) that starts
 *      on state 0 at s and ends on state S - 1 at e - 1, with spot's costs, recursion and tie rules and no fresh start after
 *      s; in exact arithmetic it is the detection's own path, in fp32 the two can part only on exact ties.  Token u's frame is
 *      the first frame of the path's run on state 2u; its token_logp is lp[frame, y_u].
 *   Edge spaces never fall inside a keyword: the spaces kept at a splice's left edge (greedy tokens in [s, e) before i0) are
 *   written just before y at frame s, and those at its right edge (in [s, e) from i1 on) whose frame is at or before the
 *   frame l of y's last token are written just after y at frame l; the other right-edge spaces keep their frames.  Every
 *   other kept greedy token keeps its frame, and the output is all tokens ordered by (frame, then: greedy tokens placed
 *   before the frame's keyword token, the keyword token, greedy tokens placed after it, each group in greedy order), so
 *   frames never decrease.  out_source[i] = k for a spliced or confirmed token, -1 for the others.  Tokens past max_out are
 *   dropped and out_counts stops at max_out; with max_out >= T (required; gam_*_greedy's width) that needs more tokens than
 *   frames, which only shared frames allow.
 *   7. Scores, when the caller passes them: out_path_logp = fp32(fp64(path_logp) + E_1 + E_2 + ...) in fp64, over the accepted
 *      splices in start order (path_rows does not change); for frame_logp (device f64 [b * frame_pitch + t], the per-frame
 *      sums of gam_*_greedy_resume), every frame t of an accepted splice gets += fp64(lp[t, l(t)]) - fp64(m[t]), l(t) the
 *      traced path's label, so segment and path confidences keep their meaning.
 * Inputs, all device: log_probs [B, T, V+1], enc_len [B], keywords [K, Umax], keyword_len [K] and det_start / det_end /
 *   det_score / det_count exactly as given to and produced by gam_ctc_spot with the same threshold and max_det; token_flags u8
 *   [V]; ids / frames [B, max_out], counts [B] (gam_*_greedy); token_logp [B, max_out] and path_logp [B] (scored greedy), or
 *   NULL together with out_token_logp / out_path_logp; frame_logp, or NULL.  Outputs: out_ids / out_frames / out_source
 *   [B, max_out] (entries past out_counts[b] are not written), out_counts [B], out_token_logp [B, max_out], out_path_logp [B];
 *   they must not alias the inputs.
 * Refused (gam_last_error): what gam_ctc_spot refuses, plus max_out < T, a missing flag table or V != num_classes - 1,
 *   frame_pitch < T and a workspace smaller than gam_ctc_bias_workspace_bytes(h, B, T, K, max_det) (which returns -1 for bad
 *   sizes or a handle without a CTC head).  The workspace holds, per recording, the sort keys of K x min(max_det, T)
 *   candidates rounded up to a power of two (16 bytes each), 72 bytes per frame (the backpointers, 32 bytes per frame, among
 *   them) and 4 bytes per keyword.  Three launches, fixed orders, no atomics, no host synchronisation: capturable in a CUDA
 *   graph. */
int64_t gam_ctc_bias_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t K, int32_t max_det);
int gam_ctc_bias(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                 const int32_t* keyword_len, int32_t K, int32_t Umax, const int32_t* det_start, const int32_t* det_end,
                 const float* det_score, const int32_t* det_count, int32_t max_det, float threshold, const uint8_t* token_flags,
                 int32_t V, const int32_t* ids, const int32_t* frames, const int32_t* counts, int32_t max_out, const float* token_logp,
                 const float* path_logp, double* frame_logp, int64_t frame_pitch, void* workspace, int64_t workspace_bytes,
                 int32_t* out_ids, int32_t* out_frames, int32_t* out_counts, int32_t* out_source, float* out_token_logp,
                 float* out_path_logp, void* stream);
/* Resumable hotwords (live streams): gam_ctc_bias over a stream whose frames arrive in consecutive calls.  Each call releases
 * the output tokens no later frame can change and leaves the rest with the caller, who holds it for the next call.  Stateless:
 * the caller keeps the held rows, greedy tokens and undecided detections between calls.
 *
 * Row b holds stream frames frame_base[b] + t, t < T_b = clamp(hi[b], 0, T): log_probs [B, T, V+1] rows, the greedy tokens
 * (ids / frames / counts, frames in stream frames, strictly increasing, in [frame_base, frame_base + T_b); token_logp or NULL),
 * and the known final detections not yet decided (det_* [B, K, max_det], stream frames, each keyword's in time order: those
 * carried out of the call before, then those gam_ctc_spot_resume emitted since).  `state` is the spot records after this
 * step's gam_ctc_spot_resume over the same frames with the same keywords and threshold.  left_boundary[b] != 0 when the held
 * range starts on a word boundary: the stream starts there, or the last greedy token before it is a space (a greedy token,
 * never a spliced one).  C = frame_base + T_b is the stream's decoded frame count.
 * Three facts make an early decision exact:
 *   1. Future candidates start at or after the horizon h.  Spot costs are <= 0 (c = lp - m exactly), so a path's score never
 *      rises, and a path that ends as a candidate (E >= tau) had v >= tau at every frame it crossed.  Every detection not yet
 *      emitted therefore starts at or after h = min(C, the pending detection's start, the start frame of every state with
 *      v >= tau in every record); NaN scores fail v >= tau, as they fail E >= tau in spot.
 *   2. gam_ctc_bias's selection (step 4) accepts a candidate only against the candidates it overlaps, so the components of
 *      the overlap graph are decided independently.
 *   3. Eligibility (step 3) reads only greedy tokens: a candidate's right boundary is known once a greedy token exists at a
 *      frame >= its end, or once the stream has finished.
 * So a component of the known detections is decided when every member ends at or before h and a greedy token exists at a
 * frame >= its last end (with finish[b], every component is).  The release frame is R = min(h, the start of every undecided
 * detection); with finish, R = C.  Every output token at a frame < R is final: splices stay inside their spans, left-edge
 * spaces move to s and right-edge spaces to the keyword's last frame, before e.
 * Outputs: out_ids / out_frames (stream frames) / out_source / out_token_logp [B, max_out] and out_counts [B], the released
 *   tokens (frames < R) exactly as gam_ctc_bias writes them; released_until [B] = R (stream frame); carry_* [B, K, max_det] /
 *   carry_count [B, K], the detections not decided, in their order, for the next call; frame_logp (f64 [b * frame_pitch + t],
 *   the held frames' per-frame sums, or NULL) adjusted in place at the released spliced frames as gam_ctc_bias adjusts it
 *   (fp64(lp) - fp64(m), added in the same order).  The caller keeps the greedy tokens and rows at frames >= R and the carried
 *   detections.  Outputs must not alias the inputs.
 * Equality: splitting a stream's frames into consecutive calls, the last one with finish, and concatenating the released
 *   tokens gives gam_ctc_bias's ids, frames, sources, token_logp and frame_logp adjustments over the whole stream, bit for bit.
 * Held span: [R, C) is bounded by the oldest live hotword path with v >= tau, not by the stream's length; a partial path can
 *   survive a long silence, where blank costs 0.
 * Precondition, as for gam_ctc_bias: the held greedy frames are strictly increasing and lie in [frame_base, frame_base + T_b).
 *   They are device data, so the call cannot refuse other frames without a host synchronisation; a token outside the held
 *   range is never used to write outside the workspace or the outputs, but the output is then unspecified.
 * Refused (gam_last_error): what gam_ctc_bias refuses, plus a NULL hi, frame_base, finish, left_boundary, state,
 *   released_until or carry_* pointer, and a record_bytes other than gam_ctc_spot_state_bytes(h, Umax).  The workspace is
 *   gam_ctc_bias's (gam_ctc_bias_resume_workspace_bytes).  Three launches, fixed orders, no atomics, no host
 *   synchronisation, capturable in a CUDA graph; a stream's outputs do not depend on its batch or the keyword order. */
int64_t gam_ctc_bias_resume_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t K, int32_t max_det);
int gam_ctc_bias_resume(gam_handle* h, const float* log_probs, int32_t B, int32_t T, const int32_t* hi, const int32_t* frame_base,
                        const int32_t* finish, const int32_t* keywords, const int32_t* keyword_len, int32_t K, int32_t Umax,
                        const void* state, int64_t record_bytes, const int32_t* det_start, const int32_t* det_end,
                        const float* det_score, const int32_t* det_count, int32_t max_det, float threshold,
                        const uint8_t* token_flags, int32_t V, const int32_t* ids, const int32_t* frames, const int32_t* counts,
                        const int32_t* left_boundary, int32_t max_out, const float* token_logp, double* frame_logp,
                        int64_t frame_pitch, void* workspace, int64_t workspace_bytes, int32_t* out_ids, int32_t* out_frames,
                        int32_t* out_counts, int32_t* out_source, float* out_token_logp, int32_t* released_until,
                        int32_t* carry_start, int32_t* carry_end, float* carry_score, int32_t* carry_count, void* stream);
/* RNN-T stage 1: enc [B, T, d_model], dec [B, U+1, pred_hidden] (gam_rnnt_predict over cat[blank, y]), targets [B, U] i32
 *   -> blank [B, T, U+1], label [B, T, U+1]: bit-identical to the matching entries of gam_rnnt_joint's lattice for the same
 *   enc / dec, but no [.., V+1] row is ever stored.  label is -inf at u = U and NaN where targets[b, u] is outside [0, V) (so
 *   that utterance's alignment is NaN).  Workspace: the two projections, as gam_rnnt_joint's. */
int64_t gam_rnnt_align_scores_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_align_scores(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, int32_t B, int32_t T, int32_t U,
                          void* workspace, int64_t workspace_bytes, float* blank, float* label, void* stream);
/* RNN-T stage 2: blank / label [B, T, U+1] (stage 1's, or any caller scores), enc_len [B], target_len [B], all device. */
int64_t gam_rnnt_align_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_align(gam_handle* h, const float* blank, const float* label, const int32_t* enc_len, const int32_t* target_len, int32_t B,
                   int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                   float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream);

/* ---- backward passes of the three head calls above, for training the heads on a frozen encoder.  fp32, stream-ordered, no
 * host synchronisation and no atomics: every sum runs in an order fixed by the sizes, so two calls on the same inputs give
 * bit-identical gradients.  They use the handle's current head weights.  Every output pointer may be NULL (not computed),
 * except that a weight gradient and its bias gradient go together.  Each needs a workspace of *_workspace_bytes().
 *
 * CTC: grad = dL/dlog_probs [B, T, V+1], log_probs = gam_ctc_log_probs's output.  dlogit = grad - exp(log_probs) * rowsum(grad);
 *   d_enc [B, T, d_model] = dlogit W, dW [V+1, d_model] = sum over frames of dlogit^T enc, db [V+1] = sum of dlogit. */
int64_t gam_ctc_log_probs_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T);
int gam_ctc_log_probs_backward(gam_handle* h, const float* enc, int32_t B, int32_t T, const float* log_probs, const float* grad,
                               void* workspace, int64_t workspace_bytes, float* d_enc, float* dW, float* db, void* stream);
/* Joint: grad [B, T, U, V+1], log_probs = gam_rnnt_joint's output.  The hidden rows relu(E[b,t] + P[b,u]) are rebuilt from the
 * two projections, never stored; their gradient dhid [B, T, U, joint_hidden] is kept in the workspace.  Outputs: d_enc
 * [B, T, d_model], d_dec [B, U, pred_hidden], and the gradients of joint.enc (dW_enc [J, d_model], db_enc [J]), joint.pred
 * (dW_pred [J, pred_hidden], db_pred [J]) and joint.joint_net.1 (dW_out [V+1, J], db_out [V+1]).  64-bit offsets. */
int64_t gam_rnnt_joint_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_joint_backward(gam_handle* h, const float* enc, const float* dec, int32_t B, int32_t T, int32_t U, const float* log_probs,
                            const float* grad, void* workspace, int64_t workspace_bytes, float* d_enc, float* d_dec, float* dW_enc,
                            float* db_enc, float* dW_pred, float* db_pred, float* dW_out, float* db_out, void* stream);
/* Prediction LSTM: BPTT over the U steps of gam_rnnt_predict_train (x, h0, c0 as given to it; g and c_seq its outputs), one
 * launch per step.  grad_g [B, U, H] is required, grad_h1 / grad_c1 [B, H] may be NULL (zero).  embed [V+1, H], w_ih [4H, H],
 * w_hh [4H, H] are the module's lstm / embed weights (w_hh must match the packed one).  Outputs: d_h0, d_c0 [B, H]; d_embed
 * [V+1, H] with a zero blank row (nn.Embedding's padding_idx); dW_ih, dW_hh [4H, H]; d_bias [4H], the gradient of both
 * bias_ih_l0 and bias_hh_l0.  An utterance with an id outside [0, V] gets NaN in its d_h0 / d_c0 (and the weight gradients it
 * feeds).  pred_hidden <= GAM_PREDICT_BACKWARD_MAX_HIDDEN. */
int64_t gam_rnnt_predict_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t U);
int gam_rnnt_predict_backward(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, const float* g,
                              const float* c_seq, const float* grad_g, const float* grad_h1, const float* grad_c1, const float* embed,
                              const float* w_ih, const float* w_hh, void* workspace, int64_t workspace_bytes, float* d_h0, float* d_c0,
                              float* d_embed, float* dW_ih, float* dW_hh, float* d_bias, void* stream);

/* ---- fused RNN-T loss: -log p(y | x) summed over all alignments, and its gradient, without the [B, T, U+1, V+1] lattice.
 * Notation as for gam_rnnt_align: nodes (t, u), t < T_b, u <= U_b; blank(t, u) and label(t, u) are stage 1's scores
 * (gam_rnnt_align_scores, bit for bit) and lse(t, u) is the log-sum-exp of row joint(t, u) that both subtract.
 *   alpha: gam_rnnt_align's forward recursion, the same lse2 operands in the same order; ll = alpha(T_b - 1, U_b) +
 *     blank(T_b - 1, U_b) and loss[b] = -ll, so loss[b] == -log_likelihood[b] of gam_rnnt_align bit for bit
 *     (= torchaudio rnnt_loss(..., blank=V, reduction="none") on the lattice).
 *   beta: beta(T_b - 1, U_b) = blank(T_b - 1, U_b); beta(t, u) = lse2(blank(t, u) + beta(t + 1, u), label(t, u) + beta(t, u + 1)),
 *     -inf outside the lattice.
 *   edge occupancies: e_blank(t, u) = exp(alpha + blank + beta(t + 1, u) - ll), with beta(T_b, U_b) := 0 for the closing edge;
 *     e_label(t, u) = exp(alpha + label + beta(t, u + 1) - ll) for u < U_b, else 0; gamma = e_blank + e_label, defined so (not
 *     as exp(alpha + beta - ll)) that sum_v dz[v] = 0 holds as closely as fp32 allows.
 *   per-node logit gradient, upstream g = grad_loss[b]:
 *     dz[v] = g (exp(z_v - lse) gamma - [v = blank] e_blank - [v = y_{u+1}] e_label), z = W_o h + b_o, h = relu(E[b,t] + P[b,u]).
 *   back through the joint: dhid = (dz W_o) * [E + P > 0] (relu's gradient at 0 is 0, as torch's); dW_out = sum dz h^T,
 *     db_out = sum dz; dE[b, t] = sum_u dhid, dP[b, u] = sum_t dhid; then d_enc, d_dec and the projection gradients exactly as
 *     gam_rnnt_joint_backward forms them from dE / dP.
 * Edge cases: T_b = 0 gives loss +inf; an utterance whose loss is +inf (T_b = 0, or no path of finite score) contributes no
 * gradient.  U_b = 0 is the blank-only path.  A NaN in any score the recursion reads (a target id outside [0, V) makes its label
 * NaN) makes that utterance's loss NaN and puts NaN in every gradient it feeds; the other utterances' losses are untouched.
 * Nodes outside an utterance's lattice, and target entries at or past target_len[b], are never read into a result.
 *
 * Sizes: enc [B, T, d_model], dec [B, U+1, pred_hidden] (gam_rnnt_predict over cat[blank, y]), targets [B, U] i32, enc_len [B],
 * target_len [B] i32, all device.  Limits are gam_rnnt_align's (U <= 4096, T <= the handle's max_encoded_frames) plus
 * joint_hidden <= GAM_RNNT_LOSS_MAX_JOINT_HIDDEN (a multiple of 4); the *_bytes functions return -1 beyond them or for a handle without an RNN-T head.
 * Memory, N = B T (U+1) nodes, J = joint_hidden, fp32:
 *   saved (kept between the calls): 12 N bytes = [lse | e_blank | e_label], each [B, T, U+1];
 *   forward workspace: 12 N bytes (blank, label, alpha) + 4 (B T + B (U+1)) J bytes (the projections), 1 KiB-aligned pieces;
 *   backward workspace: 4 J (2 B T + 2 B (U+1) + NS B T + ST B (U+1)) bytes + max(4 S V1 (J+1), the projection gradients'
 *     partials), with NS = ceil((U+1) / 64) column strips, ST <= 64 frame ranges and S <= 64 node slices (rnnt_loss.cu's plan).
 * No atomics and every sum in a fixed order: repeated calls give bit-identical gradients, and an utterance's loss is the same
 * bits in any batch.  Stream-ordered, no host synchronisation, capturable in a CUDA graph.
 *
 * gam_rnnt_loss: -> saved (gam_rnnt_loss_saved_bytes), loss [B] f32.
 * gam_rnnt_loss_backward: the forward's enc, dec, targets, lengths and saved, grad_loss [B] f32 -> d_enc [B, T, d_model],
 *   d_dec [B, U+1, pred_hidden], dW_enc [J, d_model], db_enc [J], dW_pred [J, pred_hidden], db_pred [J], dW_out [V+1, J],
 *   db_out [V+1].  Every output may be NULL (not computed), except that a weight gradient and its bias gradient go together. */
int64_t gam_rnnt_loss_saved_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int64_t gam_rnnt_loss_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_loss(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, const int32_t* enc_len,
                  const int32_t* target_len, int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, float* saved,
                  float* loss, void* stream);
int64_t gam_rnnt_loss_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U);
int gam_rnnt_loss_backward(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, const int32_t* enc_len,
                           const int32_t* target_len, int32_t B, int32_t T, int32_t U, const float* saved, const float* grad_loss,
                           void* workspace, int64_t workspace_bytes, float* d_enc, float* d_dec, float* dW_enc, float* db_enc,
                           float* dW_pred, float* db_pred, float* dW_out, float* db_out, void* stream);

/* Emotion head  <- gigaam/model.py:272-293 (GigaAMEmo.get_probs / forward_for_export): the mean of utterance b's encoder
 * frames, logits = W mean + b, probs = softmax(logits), fp32.
 *   enc: device f32 [B, T, d_model] (gam_encode's layout); enc_len: device i32 [B], or NULL = all T frames.
 *   Frames pooled for utterance b: n_b = enc_len[b] clamped to [0, T], except that a batch of ONE pools all T frames (the
 *   rule of gam_encode's packed rows, and what the reference's get_probs does).  Frames t >= n_b are never read; n_b = 0
 *   gives a NaN row.  Utterance b's summation order depends on n_b alone, so its outputs are bit-identical in any batch.
 *   -> pooled: device f32 [B, d_model], logits / probs: device f32 [B, C]; each may be NULL (not written).
 * workspace: device scratch of at least gam_emo_workspace_bytes(B, T) bytes.  Two launches, no host synchronisation:
 * capturable in a CUDA graph.  gam_emo_workspace_bytes returns -1 for a handle without an emo head or bad sizes
 * (B < 1, T < 1 or T > 2 097 120). */
int64_t gam_emo_workspace_bytes(const gam_handle* h, int32_t B, int32_t T);
int gam_emo_head(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                 int64_t workspace_bytes, float* pooled, float* logits, float* probs, void* stream);
/* ---- Emotions over time.  The head is Linear(d_model, C) on the mean of the frames, so in real arithmetic
 * softmax(W mean_t f_t + b) = softmax(mean_t l_t) with l_t = W f_t + b: any span's emotion follows from the per-frame logits.
 *
 * gam_emo_frame_logits: enc device f32 [B, T, d_model] (gam_encode's layout); lo, hi, dst device i32 [B]; frame_logits device
 *   f32 [n_frames, C].  Row b's local frames t in [lo'[b], hi'[b]), lo' and hi' being lo[b] and hi[b] clamped to [0, T], get
 *   their logits written to row dst[b] + t - lo'[b] of frame_logits; a row outside [0, n_frames) is dropped and every other row
 *   is left as it was.  Frames outside [lo', hi') are never read.  The dot product is gam_emo_head's: per class, lane l of a
 *   warp sums k = 4 l + 128 i (i ascending) with fp32 FMAs from +0, then the xor tree 16, 8, 4, 2, 1, then + bias.  So a
 *   frame's logits have the same bits whichever batch row, window or launch produced them, and a recording's windows are
 *   stitched by one launch per batch of windows, straight into the recording's [T, C] buffer.
 * gam_emo_spans: frame_logits device f32 [n_frames, C]; span_start, span_end device i32 [S], each span [a, b) clamped to
 *   [0, n_frames] (b < a is empty) -> logits [S, C] = the mean of l over the span's n frames, probs [S, C] = its softmax; either
 *   output may be NULL (not written).  The mean sums each run of 32 frames in ascending t from its first frame, adds the run
 *   sums from +0 in ascending order and divides by n (gam_emo_head's order); the softmax is gam_emo_head's.  The order depends
 *   only on the span's length, so a span's outputs have the same bits at any position in the list, next to any other spans.
 *   An empty span gives a NaN row, the mean of an empty set.  A NaN frame logit makes that class's mean NaN in every span
 *   containing it, and with it the span's whole probs row.
 * lo, hi, dst and the spans are device data: their ranges are a precondition, not a refusal; values outside them never cause a
 * read outside enc / frame_logits or a write outside frame_logits / logits / probs.
 * Refused (gam_last_error): a handle without an emo head, B outside [1, 65535], T < 1 or n_frames < 1, S < 1, and a NULL enc,
 * lo, hi, dst, frame_logits, span_start or span_end.  One launch each, fixed orders, no atomics, no workspace, no host
 * synchronisation: capturable in a CUDA graph. */
int gam_emo_frame_logits(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi, const int32_t* dst,
                         float* frame_logits, int32_t n_frames, void* stream);
int gam_emo_spans(gam_handle* h, const float* frame_logits, int32_t n_frames, const int32_t* span_start, const int32_t* span_end,
                  int32_t S, float* logits, float* probs, void* stream);

/* Resampling to 16 kHz  <- the reference resamples with ffmpeg (-ar 16000, gigaam/preprocess.py:12-40); this is torchaudio's
 * default resample(x, orig, 16000) (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), restated:
 *   g = gcd(orig, 16000), o = orig / g, n = 16000 / g, base = min(o, n) * 0.99, w = ceil(6 o / base) (double arithmetic),
 *   K = 2 w + o taps.  h[p, k], p in [0, n), k in [0, K): torchaudio's _get_sinc_resample_kernel evaluated in float64 and
 *   rounded once to fp32 (built on the host: preprocess.resample_table).
 *   y[j n + p] = sum_k h[p, k] x[j o + k - w], samples outside the signal 0; the sum runs over k in increasing order as one
 *   chain of fp32 FMAs from +0 (skipping taps whose sample is outside the signal gives the same bits), so every output is a
 *   function of its own taps only.  A signal of len samples gives ceil(n len / o) outputs (integer arithmetic).
 *   orig = 16000 is not resampled: callers make no launch and build no table.
 *
 * gam_resample: a ragged batch of B rows.  spans: device i64 [4, B] = in_begin, in_end, out_begin, out_end; row b of x
 *   (device f32, row pitch x_pitch) holds the samples [in_begin[b], in_end[b]) of its signal from column 0 (at most x_pitch of
 *   them are read), every other sample counts as 0; row b of y (device f32, row pitch y_pitch) gets outputs
 *   [out_begin[b], out_end[b]) from column 0, at most y_pitch of them.  Nothing else of y is written: a row whose out range is
 *   empty or inverted writes nothing, and an inverted in range reads nothing (Engine.resample refuses both on the host).  The
 *   one-shot case is in = [0, len), out = [0, ceil(n len / o)); chunks and streams pass the spans of their pieces.
 *   table: device f32 [table_rows, table_cols] = [2 w + o, n], h transposed (k-major).  One launch, no atomics, no host synchronisation, capturable in a
 *   CUDA graph.  Refused (gam_last_error): a NULL pointer, B outside [1, 65535], a negative pitch, n or o < 1, table dimensions
 *   other than [2 w + o, n] for (o, n), and tables of more than 2^20 entries. */
int gam_resample(gam_handle* h, const float* x, int64_t x_pitch, int32_t B, const int64_t* spans, const float* table,
                 int32_t table_rows, int32_t table_cols, int32_t o, int32_t n, float* y, int64_t y_pitch, void* stream);

/* ---- the one multi-GPU exchange of the path (SURVEY 8e): utterances are sharded over ranks, one process per GPU, and the
 * device-resident hypotheses are all-gathered ONCE over NCCL (NVLink / NVSwitch) when the batch was actually split.
 * gam_comm_unique_id: rank 0 fills 128 bytes, the host ships them to every rank by any channel (torch.distributed, MPI,
 * a file); gam_comm_init: collective over all ranks, binds an NCCL communicator to the handle; gam_gather_hyps: every
 * rank passes ONE packed int32 device buffer [ids B_local x W | frames B_local x W | counts B_local] of n_int32 elements
 * (same n on every rank: pad short shards with counts = 0) and receives gathered[r * n_int32 ...] = rank r's buffer.
 * Stream-ordered, capturable in a CUDA graph, no host synchronisation.  NCCL is bound at run time (dlopen): hosts without
 * it keep every other entry point; these three then return an error. */
int gam_comm_unique_id(uint8_t* out128);
int gam_comm_init(gam_handle* h, const uint8_t* id128, int32_t rank, int32_t nranks);
int32_t gam_comm_nccl_version(void);
int gam_gather_hyps(gam_handle* h, const int32_t* packed, int64_t n_int32, int32_t* gathered, void* stream);

/* Word grouping of hypotheses on the device  <- gigaam/timestamps_utils.py:13-53 frames_to_words (gigaam/model.py:104-124).
 * ids / frames / counts as produced by gam_*_greedy (row pitch max_out); token_flags: device u8 [V], bit 0 = the piece is
 * " " (delimiter), bit 1 = the piece starts with U+2581 (opens a new word), bit 2 = the piece (prefix removed) is empty
 * after strip().  Per utterance b and word w < n_words[b] (row pitch max_words; max_words >= max_out is always enough):
 * word_start = frame of the first piece, word_end = frame of the last piece + 1, and the pieces are tokens
 * [word_first_token, word_first_token + word_tokens) of ids[b].  Times = frame * frame_shift on the host. */
int gam_group_words(gam_handle* h, const int32_t* ids, const int32_t* frames, const int32_t* counts, int32_t B, int32_t max_out,
                    const uint8_t* token_flags, int32_t V, int32_t max_words, int32_t* word_start, int32_t* word_end,
                    int32_t* word_first_token, int32_t* word_tokens, int32_t* n_words, void* stream);

/* ---- unit entry points (parity tests of the individual kernels).  Operands come from the caller, not from the handle; every
 * size the kernel does not support is refused, and device-side row maps are read back and checked against the buffers
 * (these calls synchronise the stream to do so: they are for tests, not for the hot path). ---- */
/* D[M,N] = A[M,K] W[N,K]^T with epilogue `kind` (0 bias->f16, 1 bias+silu->f16, 2 bias+glu->f16 [N/2 cols],
 * 3 res + scale*(acc+bias) -> f32, 4 bias -> f32, 7 DFT power (re^2 + im^2) * 2^-28 -> f32 [N/2 cols], no bias), written to
 * columns [col0, col0 + cols) of out (and read from the same columns of res; res == out is allowed) with row pitch ldo.
 * A2 != NULL (kind 0 only): columns [0, n1) read A, [n1, N) read A2 (one launch, as gam_encode's q/k/v projection).
 * reverse: walk the tiles from the last; m_dev: device i32 row count (clamped to [0, M]; rows at or past it are not written)
 * or NULL = M.  A, A2, W fp16 device [M or N, K]; N % 256 == 0; K % 64 == 0. */
int gam_test_gemm(gam_handle* h, int32_t kind, const void* A, const void* A2, int32_t n1, const void* W, const float* bias,
                  const float* res, void* out, int32_t M, int32_t N, int32_t K, int32_t ldo, int32_t col0, float scale,
                  int32_t reverse, const int32_t* m_dev, void* stream);
/* 1 when the last gam_test_gemm launch stored its full tiles (every row live) through shared memory and TMA bulk stores,
 * 0 when every tile was stored straight from the registers (residual and power kinds, or an output column range TMA
 * cannot address: base or row pitch not 16-byte aligned). */
int gam_test_gemm_used_slots(gam_handle* h);
/* Implicit-GEMM stride-2 convolutions of the subsampling, out[frame, N] = relu(conv + bias) for frames t < len_out[b], 0 for the
 * others (fp16, or fp32 when f32_out):
 *   conv1d == 0: 3x3 / pad 1 over channels-last A f16 [B, T_in, F1 = 32, C], W = [N, (kt, kf, c)] f16; frame row = 16 rows
 *                (one per output bin) of out [out_frames * 16, N];
 *   conv1d == 1: `taps` / pad (taps-1)/2 over time-major A f16 [B, T_in, C], W = [N, (tap, c)] f16; out [out_frames, N].
 * T_out = floor((T_in + 2 pad - k) / 2 + 1).  cu / plen (device i32 [B], both or neither): frame (b, t < plen[b]) -> row cu[b] + t
 * and nothing else is written; NULL: frame (b, t) -> row b * T_out + t for every t < T_out. */
int gam_test_gemm_conv(gam_handle* h, int32_t conv1d, const void* A, const void* W, const float* bias, const int32_t* len_out,
                       const int32_t* cu, const int32_t* plen, void* out, int32_t out_frames, int32_t B, int32_t T_in, int32_t F1,
                       int32_t C, int32_t taps, int32_t N, int32_t f32_out, void* stream);
/* LayerNorm(768, eps 1e-5) of fp32 rows -> fp16, rows at or past *rows_dev (NULL: rows) untouched; reverse walks them from the last */
int gam_test_layernorm(gam_handle* h, const float* x, const float* g, const float* b, void* out, int32_t rows, const int32_t* rows_dev,
                       int32_t reverse, void* stream);
/* LayerNorm + rotary embedding: out_u = LN(x) f16, out_r = rope(LN(x)) f16 per head of 2*half_dim with the [table_rows, half_dim]
 * fp32 cos / sin tables at position row_t[row] (device i32, or NULL: row % T) */
int gam_test_ln_rope(gam_handle* h, const float* x, const float* g, const float* b, const float* rope_cos, const float* rope_sin,
                     int32_t table_rows, int32_t half_dim, void* out_u, void* out_r, int32_t rows, const int32_t* rows_dev,
                     const int32_t* row_t, int32_t T, int32_t reverse, void* stream);
/* x_out = LN_out(r) fp32 (x_out may be r), y_out = LN_next(x_out) f16 (y_out NULL: not computed) */
int gam_test_ln_out_ln(gam_handle* h, const float* r, const float* g_out, const float* b_out, const float* g_next, const float* b_next,
                       float* x_out, void* y_out, int32_t rows, const int32_t* rows_dev, int32_t reverse, void* stream);
/* packed fp32 rows x [rows, 768] -> out f32 [B, T, 768]: out[b, t] = x[cu[b] + t] (LayerNorm'd when gamma != NULL) for
 * t < plen[b], zeros elsewhere */
int gam_test_unpack_rows(gam_handle* h, const float* x, const float* gamma, const float* beta, const int32_t* cu, const int32_t* plen,
                         float* out, int32_t B, int32_t T, int32_t rows, int32_t reverse, void* stream);
/* depthwise conv (kw = 5 or 31 taps, w f32 [kw, 768], frames t >= len[b] read as zero) + SiLU, layer_norm == 0: bias carries the
 * folded BatchNorm; layer_norm == 1: LayerNorm over channels (gamma, beta) before the SiLU.  g, out f16 [rows, 768]: utterance
 * b at row cu[b] with plen[b] frames (cu / plen NULL: row b * T, T frames); the LayerNorm variant walks rows < *rows_dev (NULL:
 * B * T) and finds their (utterance, frame) in row_b / row_t when packed. */
int gam_test_dwconv(gam_handle* h, int32_t layer_norm, const void* g, const float* w, const float* bias, const float* gamma,
                    const float* beta, const int32_t* len, const int32_t* cu, const int32_t* plen, const int32_t* row_b,
                    const int32_t* row_t, const int32_t* rows_dev, void* out, int32_t B, int32_t T, int32_t rows, int32_t kw,
                    void* stream);
/* gam_encode's first kernels: stage lengths of the subsampling (kernel size k) for mel lengths mel_len (device i64 [B]) and
 * M mel frames, and the packed-row plan: len0..len2, plen, run1 i32 [B], cu i32 [B + 1], rows_dev i32 [1], row_b / row_t
 * i32 [B * T'] (rows < cu[B] written) */
int gam_test_pack_plan(gam_handle* h, const int64_t* mel_len, int32_t B, int32_t k, int64_t M, int32_t* len0, int32_t* len1,
                       int32_t* len2, int32_t* plen, int32_t* run1, int32_t* cu, int32_t* rows_dev, int32_t* row_b, int32_t* row_t,
                       void* stream);
/* conv2d subsampling stage 1: mel f32 [B, F, M] -> out f16 [B, T1, F1, C] (3x3 / stride 2 / pad 1, one input channel, w f32
 * [C, 9]); mel frames >= len0 read as zero, frames >= len1 written as zero, 8-frame blocks from run1[b] on (run1 may be NULL)
 * not written */
int gam_test_subsample_conv1(gam_handle* h, const float* mel, const int32_t* len0, const int32_t* len1, const int32_t* run1,
                             const float* w, const float* bias, void* out, int32_t B, int32_t F, int64_t M, int32_t C, void* stream);
/* mel f32 [B, F, M] -> time-major f16 [B, M, F], frames >= len0[b] zeroed (conv1d subsampling input) */
int gam_test_mel_to_tmajor(gam_handle* h, const float* mel, const int32_t* len0, void* out, int32_t B, int32_t F, int64_t M, void* stream);
/* gam_logmel_tc's first stage: wav f32 [B, n_samples] -> A' f16 [B * M, 3 Kp] = [hi | lo | hi] of the windowed frames x 2^e_f
 * (Kp = n_fft rounded up to 64, columns [n_fft, Kp) zero) and fexp i32 [B * M] = e_f (11 unless a hi would overflow) */
int gam_test_frames_split(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, void* A, int32_t* fexp, void* stream);
/* gam_logmel_tc's last stage: power rows P f32 [B * M, 256] of frames stored at 2^fexp (device i32 [B * M]) -> mel f32
 * [B, n_mels, M] = log(clamp(2^(22 - 2 fexp) P[:, :nbins] . fb, 1e-9, 1e9)), NaN kept; fb f32 [nbins, n_mels], mel m summed over
 * bins [mel_lo[m], mel_hi[m]) only (device i32 [n_mels]) */
int gam_test_mel_log(gam_handle* h, const float* P, const int32_t* fexp, int32_t B, int32_t M, int32_t nbins, const float* fb,
                     const int32_t* mel_lo, const int32_t* mel_hi, int32_t n_mels, float* mel, void* stream);
/* gam_rnnt_greedy's cluster kernel on caller weights (H = 320, blank = V1 - 1): encproj f32 [B, T, 320] (joint.enc applied),
 * len i32 [B], emb_gates f32 [V1, 1280] (embed W_ih^T + b_ih + b_hh), whhT f32 [320, 1280], wpT f32 [320, 320], bp [320],
 * wo f32 [V1, 320], bo [V1] -> ids / frames i32 [B, max_out], counts i32 [B].  plan (host i32 [7], or NULL) receives the
 * launch chosen: NH, GLOB, class rows per CTA in shared memory, classes per CTA, utterances per group, groups, clusters. */
int gam_test_rnnt_greedy(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                         const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                         int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts, int32_t* plan,
                         void* stream);
/* the scored twin of gam_test_rnnt_greedy (gam_rnnt_greedy_scored's kernel); plan as there */
int gam_test_rnnt_greedy_scored(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                                const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                                int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts,
                                float* token_logp, float* path_logp, int32_t* path_rows, int32_t* plan, void* stream);
/* gam_rnnt_greedy_boost's kernel on caller weights, a fresh call over [0, len[b]) as gam_test_rnnt_greedy (scored when
 * token_logp is non-NULL, which then needs path_logp and path_rows); plan as there, its class rows per CTA in shared memory
 * already net of the bonus slices */
int gam_test_rnnt_greedy_boost(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                               const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                               int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts, float* token_logp,
                               float* path_logp, int32_t* path_rows, const int32_t* boost_next, const float* boost_bonus,
                               int32_t n_states, int32_t* plan, void* stream);
/* gam_ctc_align_long with the cluster size forced to cluster_ctas (0: the library's choice), so that CTA boundaries can be
 * placed with few states; a C that leaves a CTA without states is refused.  plan (host i32 [2], or NULL) receives C and the
 * states per CTA. */
int gam_test_ctc_align_long(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                            const int32_t* target_len, int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes,
                            int32_t* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int32_t* path_rows,
                            int32_t cluster_ctas, int32_t* plan, void* stream);
/* gam_ctc_align_long_gaps with the cluster size forced, as gam_test_ctc_align_long */
int gam_test_ctc_align_long_gaps(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                                 const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                                 void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp, float* viterbi_logp,
                                 float* log_likelihood, int32_t* path_rows, uint8_t* unmatched, int32_t* unmatched_rows,
                                 float* unmatched_logp, int32_t cluster_ctas, int32_t* plan, void* stream);
/* gam_ctc_align_long_skips with the cluster size forced, as gam_test_ctc_align_long */
int gam_test_ctc_align_long_skips(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                                  const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                                  float log_psi, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                                  float* viterbi_logp, float* log_likelihood, int32_t* path_rows, uint8_t* unmatched,
                                  int32_t* unmatched_rows, float* unmatched_logp, int32_t* skipped_rows, float* skip_logp,
                                  int32_t cluster_ctas, int32_t* plan, void* stream);
/* gam_ctc_spot with the keyword warps per CTA forced to warps_per_cta in [1, 32] (0: the library's choice); the outputs do
 * not depend on it. */
int gam_test_ctc_spot(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                      const int32_t* keyword_len, int32_t K, int32_t Umax, float threshold, int32_t max_det, int32_t* det_start,
                      int32_t* det_end, float* det_score, int32_t* det_count, int32_t warps_per_cta, void* stream);
/* qkv: f16 [B*T, 3*d_model]; klen i32 [B] or NULL -> out f16 [B*T, d_model].  T up to the handle's max_encoded_frames */
int gam_test_attention(gam_handle* h, const void* qkv, const int32_t* klen, void* out, int32_t B, int32_t T, void* stream);
/* rel_pos variant: qkv f16 [B*T, 4*d_model] = [q+u | q+v | k | v]; pos f16 [2*max-1, d_model] laid out like pos_proj
 * (max = the handle's max_encoded_frames, GAM_REL_POS_MAX_T by default) */
int gam_test_attention_relpos(gam_handle* h, const void* qkv, const void* pos, const int32_t* klen, void* out, int32_t B,
                              int32_t T, void* stream);
/* packed-row (varlen) form of the two calls above, the one gam_encode uses: qkv f16 [rows, 3*d_model] (pos == NULL, rotary)
 * or [rows, 4*d_model] (pos != NULL, rel_pos); utterance b owns rows cu[b] .. cu[b] + klen[b] (cu: i32 [B + 1], klen: i32
 * [B], klen[b] <= T) -> out f16 [rows, d_model]; rows that belong to no utterance are left untouched.  This is the
 * cu_seqlens contract of flash_attn_varlen_func in gigaam/utils.py:103-155 (apply_masked_flash_attn). */
int gam_test_attention_varlen(gam_handle* h, const void* qkv, const void* pos, const int32_t* klen, const int32_t* cu, void* out,
                              int32_t B, int32_t T, int32_t rows, void* stream);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t gam_launch_count(const gam_handle* h);

/* Optional per-launch timing with CUDA events on the launching stream (bench.py's roofline leg).
 * gam_profile_begin() arms it; every kernel launched through this handle until gam_profile_end() is bracketed
 * by an event pair; gam_profile_end() synchronises the events and returns summed milliseconds and launch
 * counts per kernel class (gam_profile_class_name()).  Must not be armed during CUDA-graph capture. */
int gam_profile_begin(gam_handle* h);
int gam_profile_end(gam_handle* h, double* ms_per_class, int64_t* launches_per_class, int32_t n_classes);
int gam_profile_class_count(void);
const char* gam_profile_class_name(int32_t cls);

#ifdef __cplusplus
}
#endif
#endif /* GIGAAM_B200_H_ */
