// Internal launcher declarations shared by the translation units of libgigaam_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace gam {

// rowops.cu
// Rows are packed: `rows` is the padded maximum the grid is sized for, `rows_dev` (may be null) the live count on the device.
// `reverse`: walk the rows from the last to the first (see GemmParams::reverse: consecutive kernels alternate direction)
void launch_ln_f16(const float* x, const float* g, const float* b, __half* out, int rows, const int* rows_dev, int reverse,
                   cudaStream_t s);
// row_t (may be null: row % T): frame index of every packed row inside its utterance = its rotary position
void launch_ln_rope_f16(const float* x, const float* g, const float* b, const float* rope_cos, const float* rope_sin,
                        __half* out_u, __half* out_r, int rows, const int* rows_dev, const int* row_t, int T, int half_dim,
                        int reverse, cudaStream_t s);
void launch_ln_out_ln(const float* r, const float* g_out, const float* b_out, const float* g_next, const float* b_next,
                      float* x_out, __half* y_out, int rows, const int* rows_dev, int reverse, cudaStream_t s);
// packed fp32 rows -> padded [B, T, 768] (LayerNorm on the way when gamma != null); frames that do not exist become zeros
void launch_unpack_rows(const float* x, const float* gamma, const float* beta, const int* cu, const int* plen, float* out, int B,
                        int T, int reverse, cudaStream_t s);
// cu / plen null: padded layout (utterance b at row b*T, T rows)
int launch_dwconv_bn_silu(const __half* g, const float* w, const float* bias, const int* len, const int* cu, const int* plen,
                          __half* out, int B, int T, int kw, cudaStream_t s);
int launch_dwconv_ln_silu(const __half* g, const float* w, const float* bias, const float* gamma, const float* beta,
                          const int* len, const int* cu, const int* row_b, const int* row_t, const int* rows_dev, __half* out,
                          int B, int T, int kw, cudaStream_t s);
// stage lengths of the subsampling + the packed-row plan (plen, cu [B+1], rows_dev [1], run1, row -> (b, t) maps)
void launch_pack_plan(const long long* mel_len, int B, int pad2_minus_k, int max_T0, int T1, int T2, int* len0, int* len1,
                      int* len2, int* plen, int* run1, int* cu, int* rows_dev, int* row_b, int* row_t, cudaStream_t s);

// frontend.cu
int launch_logmel(const float* wav, int B, int n_samples, int n_frames, const float* window, const float* tcos,
                  const float* tsin, const float* fb, float* mel, int n_fft, int hop, int center, int n_mels,
                  cudaStream_t s);
// run1 (may be null): stage-1 frames per utterance that are produced at all (pack_plan_kernel)
int launch_subsample_conv1(const float* mel, const int* len0, const int* len1, const int* run1, const float* w, const float* bias,
                           __half* out, int B, int M, int F, int T1, int F1, int C, cudaStream_t s);

// attention_sm90.cu
// klen (may be null: T): keys / queries of utterance b that exist; cu (may be null): packed rows, utterance b starts at row
// cu[b] and only its klen[b] query rows are computed and stored (null: row b*T, all T query rows stored)
int launch_attention(const CUtensorMap* tmap_qkv, const int* klen, const int* cu, __half* out, int B, int T, int H, int dk,
                     int d_model, cudaStream_t s);

// attention_relpos_sm90.cu: qkv [B*T, 4*d_model] = [q+u | q+v | k | v]; pos = projected position table of 2*max_t-1 rows,
// row max_t-1-r for relative position r; T <= max_t
int launch_attention_relpos(const CUtensorMap* tmap_qkv, const CUtensorMap* tmap_pos, int max_t, const int* klen, const int* cu,
                            __half* out, int B, int T, int H, int dk, int d_model, cudaStream_t s);

// ctc.cu: labels [R] of every row; lp (or NULL: unscored) [R] f32 scratch of each row's log_softmax(row)[label]
void launch_ctc_argmax(const float* enc, const float* W, const float* bias, int* labels, float* lp, int R, int D, int V1,
                       cudaStream_t s);

// Resumable greedy decoding (gam_*_greedy_resume): what the greedy loop keeps across a frame boundary, one record per decoding
// stream.  CTC uses the record up to `h`; RNN-T all of it.  A fresh utterance is label = blank, pending = 1, zeros elsewhere.
constexpr int kDecodeStateH = 320;
struct alignas(16) DecodeState {
  int label;        // CTC: the previous frame's label; RNN-T: the last label fed to the prediction network
  int pending;      // RNN-T: that label's LSTM step has not run yet
  int count;        // tokens emitted so far (the true count: not capped by max_out)
  int rows;         // decision rows so far (scored calls)
  double path;      // RNN-T: fp64 sum of l over those rows (warp 0's running sum)
  double pad;       // keeps the CTC record (up to h) a multiple of 16 bytes
  union {
    double part[32];  // CTC: the fp64 partial sums of the scored collapse, partial k over the rows r with r % 32 == k
    int boost_state;  // RNN-T: the boost graph's state (gam_rnnt_greedy_boost); 0, the initial state, in a fresh record
  };
  float h[kDecodeStateH], c[kDecodeStateH], pg[kDecodeStateH];   // RNN-T: LSTM state and W_p h + b_p
};
constexpr int64_t kCtcDecodeStateBytes = static_cast<int64_t>(offsetof(DecodeState, h));
constexpr int64_t kRnntDecodeStateBytes = static_cast<int64_t>(sizeof(DecodeState));
static_assert(kCtcDecodeStateBytes % 16 == 0, "state records stay 16-byte aligned");
static_assert(sizeof(DecodeState) == 4128 && offsetof(DecodeState, boost_state) == 32,
              "the boost state shares the CTC partial sums' bytes; the RNN-T record keeps its size");
void launch_decode_state_init(uint8_t* state, int64_t stride, int n, int blank, cudaStream_t s);

// What a greedy decode of B streams writes, and which frames of each stream it decodes (launch_ctc_collapse,
// launch_rnnt_greedy).  A fresh call (state NULL) decodes frames [0, hi[b]) of row b from a fresh stream, emits frames t and
// writes counts (and, scored, path_logp / path_rows) for every row; lo and frame_base are not read.  A resume call continues
// the DecodeState at state + b * stride over frames [lo[b], hi[b]), appends at counts[b], emits frames frame_base[b] + t and
// stores the record back; a row with lo[b] == hi[b] keeps its record and outputs.  Either way decoding [0, L) of a stream in
// consecutive calls gives a fresh call's bits.
struct GreedyIo {
  int* ids;              // [B, max_out]
  int* frames;           // [B, max_out]
  int* counts;           // [B]: tokens stored (at most max_out)
  int max_out;
  float* token_logp;     // [B, max_out]; NULL: unscored, and the three score outputs are not written
  float* path_logp;      // [B] sum of l over the decision rows (scored)
  int* path_rows;        // [B] their number (scored)
  double* frame_logp;    // [b * frame_pitch + frame] sum of l over the frame's decision rows (scored), or NULL
  int* frame_rows;       // [b * frame_pitch + frame] their number (set with frame_logp)
  int64_t frame_pitch;
  const int* lo;         // [B] (resume)
  const int* hi;         // [B] one past the last frame: the lengths for a fresh call
  const int* frame_base; // [B] (resume)
  uint8_t* state;        // DecodeState records, or NULL: a fresh call
  int64_t stride;
};
// CTC collapse of labels [B, T] (lp [B, T] from launch_ctc_argmax when scored)
void launch_ctc_collapse(const int* labels, const float* lp, int B, int T, int blank, const GreedyIo& io, cudaStream_t s);

// words.cu: (token id, frame) pairs -> word records (first frame, last frame + 1, first token, tokens) per utterance
void launch_group_words(const int* ids, const int* frames, const int* counts, const unsigned char* flags, int B, int V, int max_out,
                        int max_words, int* w_start, int* w_end, int* w_first, int* w_ntok, int* n_words, cudaStream_t s);

// resample.cu: gam_resample's polyphase resampler.  table f32 [K, n] (k-major), spans i64 [4, B] = in_begin, in_end,
// out_begin, out_end; row b of x holds samples [in_begin, in_end) and row b of y gets outputs [out_begin, out_end), both
// from column 0.  B <= 65535.
void launch_resample(const float* x, int64_t x_pitch, const float* table, int n, int o, int w, int K, const int64_t* spans, int B,
                     float* y, int64_t y_pitch, cudaStream_t s);

// rnnt.cu
// C[M,N] = A[M,K] W[N,K]^T + bias (bias may be null); K % 16 == 0
void launch_sgemm_tn_bias(const float* A, const float* W, const float* bias, float* C, int M, int N, int K, cudaStream_t s);
// the same with W given transposed: Wt[K,N] row-major, N % 4 == 0
void launch_sgemm_nn_bias(const float* A, const float* Wt, const float* bias, float* C, int M, int N, int K, cudaStream_t s);

// pooled_head.cu: GigaAMEmo's head.  enc f32 [B, T, 768], enc_len i32 [B] or null -> part f32 [B, pool_chunk_count(T), 768]
// (sums of kPoolChunk frames; chunks past an utterance's length are not written), then pooled [B, 768] = mean over the
// utterance's frames, logits [B, C] = W pooled + b, probs [B, C] = softmax(logits); any of the three may be null.  Frames pooled
// for utterance b: enc_len[b] clamped to [0, T], or all T for B == 1 or enc_len == null.  1 <= C <= kPoolMaxClasses,
// 1 <= B, 1 <= T, pool_chunk_count(T) <= 65535.
constexpr int kPoolChunk = 32;
constexpr int kPoolMaxClasses = 256;
inline int pool_chunk_count(int T) { return (T + kPoolChunk - 1) / kPoolChunk; }
void launch_pool_chunks(const float* enc, const int* enc_len, int B, int T, float* part, cudaStream_t s);
void launch_pooled_head(const float* part, const int* enc_len, int B, int T, const float* W, const float* bias, int C, float* pooled,
                        float* logits, float* probs, cudaStream_t s);

// emo_time.cu: GigaAMEmo over time.  emo_frame_logits: for each row b of enc f32 [B, T, 768], local frames t in
// [lo', hi') = [clamp(lo[b], 0, T), clamp(hi[b], 0, T)) -> frame_logits row dst[b] + t - lo' ([n_frames, C]; rows outside [0, n_frames)
// are dropped) = W enc[b, t] + bias in pooled_head_kernel's order.  emo_spans: spans [a_i, b_i) of frame_logits, clamped to
// [0, n_frames] -> logits [S, C] (the mean) and probs [S, C] (its softmax), either may be null.  lo / hi / dst / spans are
// device i32.  1 <= C <= kPoolMaxClasses, 1 <= B <= 65535, 1 <= S.
void launch_emo_frame_logits(const float* enc, int B, int T, const int* lo, const int* hi, const int* dst, const float* W,
                             const float* bias, int C, float* frame_logits, int n_frames, cudaStream_t s);
void launch_emo_spans(const float* frame_logits, int n_frames, int C, const int* span_start, const int* span_end, int S, float* logits,
                      float* probs, cudaStream_t s);

// heads.cu: the heads' forward passes (fp32).  ctc: enc [R, D] -> log_probs [R, V1]
void launch_ctc_log_probs(const float* enc, const float* W, const float* bias, float* out, int R, int D, int V1, cudaStream_t s);
// E [B*T, J], P [B*U, J] -> out [B, T, U, V1] = log_softmax(Wo relu(E[b,t] + P[b,u]) + bo); 64-bit offsets.
// Returns 0 ok, 1 = unsupported J (J % 4 != 0 or J > rnnt_joint_max_hidden()) or grid, <0 = attribute error
constexpr size_t kJointMaxSmem = 200 * 1024;
int rnnt_joint_max_hidden();
int launch_rnnt_joint(const float* E, const float* P, const float* Wo, const float* bo, float* out, int B, int T, int U, int J,
                      int V1, cudaStream_t s);
// the same rows, but only blank [B, T, U1] and label [B, T, U1] = the log-probs of blank and of targets[b, u] (targets [B, U1 - 1]);
// lse [B, T, U1], when not null, also receives each row's log-sum-exp
int launch_rnnt_joint_gather(const float* E, const float* P, const float* Wo, const float* bo, const int* targets, float* blank,
                             float* label, float* lse, int B, int T, int U1, int J, int V1, cudaStream_t s);
// one step u of the 1-layer prediction LSTM (heads.cu: lstm_step_kernel documents the operands); H <= 1024
void launch_lstm_step(const int64_t* x, int U, int u, int V1, const float* emb_gates, const float* whh_t, const float* h_in,
                      int64_t h_pitch, const float* c_in, float* g, float* h_out, float* c_out, int B, int H, cudaStream_t s);

// align.cu: Viterbi + forward alignment over caller scores, one CTA per utterance (gam_ctc_align / gam_rnnt_align).
// bp: backpointer scratch of B * ctc_bp_words(T, U) / B * rnnt_bp_words(T, U) words.  Return 1 for U > kAlignMaxTokens.
constexpr int kAlignMaxTokens = 4096;
int64_t ctc_bp_words(int T, int U);
int64_t rnnt_bp_words(int T, int U);
int launch_ctc_align(const float* log_probs, const int* enc_len, const int* targets, const int* target_len, int B, int T, int U, int V1,
                     uint32_t* bp, int* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int* path_rows,
                     cudaStream_t s);
int launch_rnnt_align(const float* blank, const float* label, const int* enc_len, const int* target_len, int B, int T, int U, uint32_t* bp,
                      int* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int* path_rows, cudaStream_t s);
// rnnt_loss.cu: the fused RNN-T loss (gam_rnnt_loss / gam_rnnt_loss_backward).  Node arrays are [B, T, U + 1].
// alpha: scratch; e_blank / e_label: the edge occupancies the gradient reads; loss [B].  One CTA per utterance.
int launch_rnnt_loss_alpha_beta(const float* blank, const float* label, const int* enc_len, const int* target_len, int B, int T, int U,
                                float* alpha, float* e_blank, float* e_label, float* loss, cudaStream_t s);
// The gradient pass's grid.  Node-major: 64-node tiles of tT frames x tU lattice columns; NS column strips x ST frame ranges
// per utterance, so dE partials are [NS][B*T][J] and dP partials [ST][B*(U+1)][J].  Class-major: S node slices, partials
// [S][V1][J + 1] when S > 1.
struct RnntLossPlan {
  int tU, tT, NS, ST, S;
};
RnntLossPlan rnnt_loss_plan(int B, int T, int U, int V1);
int rnnt_loss_max_hidden();
struct RnntLossArgs {
  const float *E, *P, *Wo, *bo;   // E [B*T, J], P [B*(U+1), J] (biases included), W_o [V1, J], b_o [V1]
  const int *targets, *enc_len, *target_len;
  const float *lse, *e_blank, *e_label, *grad;
  int B, T, U, J, V1;
};
// dE_part null: no node-major pass; dW null: no class-major pass.  Returns 1 for an unsupported J, <0 on an attribute error.
int launch_rnnt_loss_grads(const RnntLossArgs& a, const RnntLossPlan& p, float* dE_part, float* dP_part, float* part, float* dW, float* db,
                           cudaStream_t s);
// the CTC sweep of launch_ctc_align over a cluster of C <= kAlignLongMaxCtas CTAs per utterance, for U <= kAlignLongMaxTokens
// and any T (gam_ctc_align_long); bp as there.  The plan is the smallest C whose states per CTA P (a multiple of 16) fit in
// shared memory at 20 bytes per state, or `forced_ctas` when it is > 0.  Return 0, 1 for a U or C that does not fit, 2 for a
// forced C that leaves a CTA without states, negative on a launch error.  plan (host, 2 ints, or NULL) receives C and P.
constexpr int kAlignLongMaxTokens = 65536;
constexpr int kAlignLongMaxCtas = 16;
constexpr int kAlignLongStaticSmem = 1024;   // headroom kept for the kernel's static shared memory
int ctc_align_long_plan(int U, int forced_ctas, int* ctas, int* states_per_cta);
// Gap mode of the sweep (gam_ctc_align_long_gaps): boundary states may also emit m[t] + log_theta.  A pre-pass fills
// m [B, T] (frames t < T_b only) before the sweep reads it.
struct AlignGaps {
  const uint8_t* line_edges;   // [B, U]: bit 0 the token starts a line, bit 1 it ends one
  float log_theta;
  float* m;                    // [B, T] workspace
  uint8_t* unmatched;          // [B, T]
  int* unmatched_rows;         // [B]
  float* unmatched_logp;       // [B]
  // skip mode (gam_ctc_align_long_skips): every line's exit blank may also be entered from the line end before it, at
  // fp32(n_i) * log_psi.  skipped_rows NULL: gap mode only.
  float log_psi;
  int* skipped_rows;           // [B]
  float* skip_logp;            // [B]
};
// gaps: NULL for gam_ctc_align_long's sweep
int launch_ctc_align_long(const float* log_probs, const int* enc_len, const int* targets, const int* target_len, int B, int T, int U,
                          int V1, int forced_ctas, uint32_t* bp, int* frames, float* token_logp, float* viterbi_logp,
                          float* log_likelihood, int* path_rows, int* plan, const AlignGaps* gaps, cudaStream_t s);

// spot.cu: CTC keyword spotting (gam_ctc_spot), grid (ceil(K / warps), B), one warp per keyword of <= kSpotMaxTokens tokens.
// keywords [K, Umax], keyword_len [K]; det_* [B, K, max_det], det_count [B, K].  log_theta = fp32 log of the threshold.
// warps: keyword warps per CTA, 1..kSpotMaxWarps, or 0 for min(kSpotWarps, K).  The plan: frames per tile (rows) and the
// dynamic shared memory of the ring.  Return 0, 1 when one tile of V1 classes does not fit in shared memory, negative on an
// attribute error.
constexpr int kSpotMaxTokens = 64;
constexpr int kSpotWarps = 8;
constexpr int kSpotMaxWarps = 32;
int ctc_spot_plan(int V1, int* rows, int* smem_bytes);
// The record of one (stream, keyword) between resume calls (gam_ctc_spot_state_bytes): this header, then each record lane's
// v[4] as f32 [4][lanes] and its start frames a[4] as i32 [4][lanes], lanes = ceil((2 Umax - 1) / 4).
struct SpotRecord {
  int has, p_start, p_end, total;   // the pending detection (when has) and the true count of detections emitted
  float p_score;
  int pad[3];
};
static_assert(sizeof(SpotRecord) == 32, "SpotRecord is one 32-byte header");
// Row b walks local frames [lo[b], hi[b]) (clamped to [0, T]) as stream frames frame_base[b] + t, from and back to its records at
// state + (b K + k) record; finish[b] != 0 emits the pending detection at the end.  state == NULL: a fresh call over [0, hi[b])
// (hi = enc_len; lo, frame_base, finish and pend_* unused).
struct SpotResume {
  const int* lo;
  const int* hi;
  const int* frame_base;
  const int* finish;
  uint8_t* state;
  int64_t record;
  int* pend_start;   // [B, K], or NULL
  int* pend_end;
  float* pend_score;
};
int64_t ctc_spot_record_bytes(int Umax);
void launch_ctc_spot_state_init(uint8_t* state, int64_t n, int Umax, cudaStream_t s);
int launch_ctc_spot(const float* log_probs, const SpotResume& io, const int* keywords, const int* keyword_len, int B, int T, int V1, int K,
                    int Umax, float log_theta, int max_det, int warps, int* det_start, int* det_end, float* det_score, int* det_count,
                    cudaStream_t s);

// bias.cu: hotwords spliced into CTC greedy output (gam_ctc_bias, gam_ctc_bias_resume), three launches in stage order 0, 1, 2: select (one CTA per
// recording), trace (kBiasTraceCtas x 4 warps per recording) and compact (one CTA per recording).  ctc_bias_workspace_words is the workspace of
// one recording in 32-bit words (a multiple of 4), or -1 when it does not fit in int64.
struct BiasArgs {
  const float* log_probs;
  const int* enc_len;
  const int* keywords;
  const int* keyword_len;
  const int* det_start;
  const int* det_end;
  const float* det_score;
  const int* det_count;
  const unsigned char* flags;
  const int* ids;
  const int* frames;
  const int* counts;
  const float* token_logp;   // nullable, with out_token_logp
  const float* path_logp;    // nullable, with out_path_logp
  double* frame_logp;        // nullable, adjusted in place, row pitch frame_pitch
  int64_t frame_pitch;
  int B, T, V1, K, Umax, max_det, max_out;
  float log_theta;
  int* out_ids;
  int* out_frames;
  int* out_counts;
  int* out_source;
  float* out_token_logp;
  float* out_path_logp;
  // gam_ctc_bias_resume; frame_base == NULL: a one-shot call (frames from 0, finished, starting on a word boundary)
  const int* frame_base;
  const int* finish;
  const int* left_boundary;
  const uint8_t* state;      // the spot records [B, K, record]
  int64_t record;
  int* released_until;
  int* carry_start;
  int* carry_end;
  float* carry_score;
  int* carry_count;
};
constexpr int kBiasTraceCtas = 32;
int64_t ctc_bias_workspace_words(int T, int K, int max_det);
void launch_ctc_bias(const BiasArgs& a, int32_t* workspace, int stage, cudaStream_t s);

// head_grads.cu: backward passes of the heads (fp32, deterministic, no atomics).  Rows are 64-bit.
// dl = G - exp(logp) * rowsum(G), rows of V1
void launch_softmax_grad(const float* G, const float* logp, float* dl, int64_t rows, int V1, cudaStream_t s);
// dW[N, K] = sum_r A[r, n] X(r, k) and, when db != null, db[n] = sum_r A[r, n]; ws: outer_sum_workspace_floats() floats.
// X(r, k): X[r, k] (plain); shift: X[r-1, k] for r % U != 0, else X0[r / U, k] (X0 null: 0); joint: relu(E[r/U] + P[bu]),
// bu = (r / U) / T * U + r % U (NaN kept)
int64_t outer_sum_workspace_floats(int64_t rows, int N, int K, bool with_bias);
void launch_outer_sum(const float* A, const float* X, int64_t rows, int N, int K, float* dW, float* db, float* ws, cudaStream_t s);
void launch_outer_sum_shift(const float* A, const float* X, const float* X0, int U, int64_t rows, int N, int K, float* dW, float* db,
                            float* ws, cudaStream_t s);
void launch_outer_sum_joint(const float* A, const float* E, const float* P, int T, int U, int64_t rows, int N, int K, float* dW,
                            float* db, float* ws, cudaStream_t s);
// out[r, k] = sum_n A[r, n] W[n * sn + k * sk], times [relu(E + P)(r, k) > 0] when mask_E != null (joint row map as above)
void launch_head_matmul(const float* A, const float* W, int64_t sn, int64_t sk, float* out, int64_t rows, int N, int K,
                        const float* mask_E, const float* mask_P, int T, int U, cudaStream_t s);
// dW[n, k] (k < K) / db[n] (k = K) = sum over z < S (ascending) of part[z][n][k], part [S][N][Kc]
void launch_outer_sum_reduce(const float* part, int S, int N, int K, int Kc, float* dW, float* db, cudaStream_t s);
// out[g, k] = sum_{i < count} X[(g / gi) * so + (g % gi) * si + i * step, k]
void launch_segment_sum(const float* X, float* out, int64_t groups, int count, int K, int64_t gi, int64_t so, int64_t si, int64_t step,
                        cudaStream_t s);
// one BPTT step u of lstm_step_kernel (u = -1: dh0 / dc0); see lstm_bwd_step_kernel.  H <= lstm_bwd_max_hidden()
int lstm_bwd_max_hidden();
void launch_lstm_bwd_step(const int64_t* x, int U, int u, int V1, const float* emb_gates, const float* whh_t, const float* whh,
                          const float* h0, const float* c0, const float* g, const float* c_seq, const float* dG, const float* dh1,
                          float* dgates, float* dc_carry, float* dh0, float* dc0, int B, int H, cudaStream_t s);
// out [V1, H4]: per-class sums of dgates rows (blank row zero); returns 1 if H4 is too large
int launch_class_gate_sum(const int64_t* x, int64_t rows, const float* dgates, int H4, int V1, int blank, float* out, cudaStream_t s);

// A boost graph (gam_rnnt_greedy_boost): next [S, V1] and bonus [S, V1], state 0 initial, S <= kBoostMaxStates
constexpr int kBoostMaxStates = 65536;
struct BoostGraph {
  const int* next;
  const float* bonus;
  int n_states;
};

// rnnt_cluster.cu: greedy decode of encproj [B, T, H] (see GreedyIo), boosted by `boost` unless it is NULL.  Returns 0 ok,
// 1 = 16-CTA clusters unavailable / unsupported shape, <0 error.  plan: host int[7] that receives the chosen launch (NH, GLOB,
// rows_smem, cls_per, nu, groups, clusters), or NULL.
int launch_rnnt_greedy(const float* encproj, const float* emb_gates, const float* whhT, const float* wpT, const float* bp,
                       const float* wo, const float* bo, int B, int T, int H, int V1, int blank, int max_symbols, const GreedyIo& io,
                       const BoostGraph* boost, int* plan, cudaStream_t s);

// gemm.cu
struct GemmParams;
enum GemmKind : int {
  GEMM_BIAS_F16 = 0,
  GEMM_BIAS_SILU_F16 = 1,
  GEMM_BIAS_GLU_F16 = 2,
  GEMM_BIAS_RES_F32 = 3,
  GEMM_BIAS_F32 = 4,
  GEMM_CONV_RELU_MASK_F16 = 5,
};
// 2-D operand GEMM  D[M,N] = A[M,K] W[N,K]^T with fused epilogue `kind`; N % 256 == 0, K % 64 == 0.
// m_dev: row count on the device (<= M), see GemmParams::m_dev.  tmap_out: the output's [M, ncol] columns (ncol = N, N/2 for
// GLU) at `out`, row pitch ldo (gam_api.cu: make_tmap_out).  With it, tiles whose rows are all live leave through shared
// memory and TMA bulk stores; without (null), and always for GEMM_BIAS_RES_F32, every tile is stored directly.
int launch_gemm(int kind, const CUtensorMap* tmap_a, const CUtensorMap* tmap_w, int M, int N, int K, const float* bias,
                const float* res, void* out, int ldo, float scale, int max_clusters, cudaStream_t s, int reverse = 0,
                const int* m_dev = nullptr, const CUtensorMap* tmap_out = nullptr);
// one launch for two GEMMs that share M, K, W's row space and the output buffer but read different A operands:
// columns [0, n1) from tmap_a1, [n1, N) from tmap_a2 (bias -> fp16).  
int launch_gemm_dual_a(const CUtensorMap* tmap_a1, const CUtensorMap* tmap_a2, int n1, const CUtensorMap* tmap_w, int M, int N,
                       int K, const float* bias, void* out, int ldo, int max_clusters, cudaStream_t s, int reverse = 0,
                       const int* m_dev = nullptr, const CUtensorMap* tmap_out = nullptr);
// implicit-GEMM 3x3/s2 conv over channels-last [B,T1,F1,C] (tmap_a 4-D strided), output [rows*16, N] fp16.
// cu / plen (both or neither): packed output rows, frame (b, t < plen[b]) -> row cu[b] + t; null: row b*T2 + t, all frames
int launch_gemm_conv(const CUtensorMap* tmap_a4d, const CUtensorMap* tmap_w, int B, int T2, int C, int N, const float* bias,
                     const int* len2, const int* cu, const int* plen, void* out, int ldo, int max_clusters, cudaStream_t s);
// implicit-GEMM k-tap/s2 conv1d over time-major [B,T_in,C_in] (tmap_a 3-D strided); out [B*T_out, N] fp16 or fp32
int launch_gemm_conv1d(const CUtensorMap* tmap_a3d, const CUtensorMap* tmap_w, int B, int T_out, int C_in, int taps, int N,
                       const float* bias, const int* len_out, const int* cu, const int* plen, void* out, int ldo, int f32_out,
                       int max_clusters, cudaStream_t s);
int launch_gemm_power(const CUtensorMap* tmap_a, const CUtensorMap* tmap_w, int M, int N, int K, float* out, int ldo, int max_clusters,
                      cudaStream_t s);
// tensor-core front end helpers (frontend.cu)
// tensor-core log-mel stages; fexp: i32 per frame, the power of two frame f is stored at (see frames_split_kernel)
int launch_frames_split(const float* wav, int B, int n_samples, int n_frames, const float* window, __half* A, int* fexp, int n_fft,
                        int Kp, int hop, int center, cudaStream_t s);
int launch_mel_log(const float* P, const int* fexp, int ldp, int B, int n_frames, int nbins, const float* fb, const int* mel_lo,
                   const int* mel_hi, float* mel, int n_mels, cudaStream_t s);
int gemm_init(int* max_clusters);   // per device: also the number of GEMM clusters that fit at once
// mel [B, F, M] f32 -> time-major fp16 [B, M, F] with frames >= len zeroed (conv1d subsampling input)
void launch_mel_to_tmajor_f16(const float* mel, const int* len0, __half* out, int B, int F, int M, cudaStream_t s);

// tensor maps (gam_api.cu)
int make_tmap_2d_f16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                     uint32_t box_cols);

}  // namespace gam
