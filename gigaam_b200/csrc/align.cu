// Viterbi and forward (log-sum-exp) alignment of known transcripts over caller-supplied fp32 scores
// (include/gigaam_b200.h, gam_ctc_align / gam_rnnt_align, has the definitions).  One CTA per utterance, fixed orders and no
// atomics, so an utterance's results are the same bits in any batch and on every call.
//   (1) ctc_align_kernel: walks the frames t.  Viterbi and forward values of the S = 2U + 1 states are double-buffered in
//       shared memory; each frame reads log_probs at the utterance's labels and at blank only.  Backpointers: 2 bits per
//       (t, s), packed 16 states to a word by shuffles.
//   (2) rnnt_align_kernel: walks the anti-diagonals d = t + u of the [T, U + 1] lattice; the nodes of one diagonal are
//       independent.  Every value is one fp32 add of two fp32 numbers, so the walk order does not change the bits.
//       Backpointers: 1 bit per node, 32 nodes of a diagonal to a word by ballot.
//   (3) ctc_align_long_kernel: (1) for long recordings.  One thread-block cluster of C <= 16 CTAs per utterance; CTA k
//       owns states [k P, (k + 1) P), P a multiple of 16, and keeps their labels and double-buffered values in its own
//       shared memory.  Each frame reads the two states left of its range from CTA k - 1 over distributed shared memory,
//       then one cluster barrier closes the frame.  The per-state arithmetic is (1)'s, so the results are its bits.
//       Gap mode (the GAPS instantiation, after row_max_kernel's pre-pass) lets the blank states at line edges also emit
//       m[t] + log theta; the instantiation without gaps is the kernel of gam_ctc_align_long.  Skip mode (SKIPS, on top
//       of gap mode) adds one edge per line, from the exit blank of the line before it to its own exit blank, whose source
//       may sit in any CTA of the cluster.
// All backtrack with one thread (a serial walk of T or T + U steps) and then gather token_logp with the whole CTA.
#include <algorithm>
#include <cmath>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"
#include "rowmax.cuh"

namespace gam {
namespace {

constexpr int kSkip = 1 << 30;   // ctc lab_s: the state may also be entered from s - 2 (skip mode, blank s: from e_i)
constexpr int kBound = 1 << 29;  // ctc_align_long lab_s, gap mode: a boundary state
// skip mode: an exit blank's lab_s holds its source as (CTA << kSrcIndexBits) | index, below the flag bits
constexpr int kSrcIndexBits = 16, kSrcCtaBits = 4;
static_assert(kAlignLongMaxCtas <= (1 << kSrcCtaBits), "a source CTA rank must fit in its lab_s field");
static_assert(kSrcIndexBits + kSrcCtaBits <= 29, "the source fields must stay below kBound and kSkip");

// gap mode: whether the blank state s (even) of a recording with U_b tokens is a boundary state: the first or last state, or
// the blank before a token that starts a line or after one that ends a line
__device__ __forceinline__ bool boundary_state(const uint8_t* edges, int Ub, int s) {
  const int j = s >> 1;   // the blank between tokens j - 1 and j
  return s == 0 || j == Ub || (edges[j] & 1) || (edges[j - 1] & 2);
}

// skip mode: the source e_i of the skip edge into the exit blank x_i = s (s >= 2, token s / 2 - 1 ends a line): the exit
// blank of the line end before it, or state 0.  A backward walk over line_edges, as long as the line.
__device__ __forceinline__ int skip_source(const uint8_t* edges, int s) {
  int j = (s >> 1) - 2;
  while (j >= 0 && !(edges[j] & 2)) --j;
  return 2 * (j + 1);
}

__device__ __forceinline__ float lse3(float a, float b, float c) {
  const float m = fmaxf(fmaxf(a, b), c);
  if (m == -INFINITY) return -INFINITY;
  return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

__device__ __forceinline__ float lse2(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log1pf(expf(fminf(a, b) - m));
}

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

// log_probs [B, T, V1], targets [B, U] (may be null when U == 0), bp: B * T * W words, W = ctc_bp_words(U)
__global__ void ctc_align_kernel(const float* __restrict__ log_probs, const int* __restrict__ enc_len, const int* __restrict__ targets,
                                 const int* __restrict__ target_len, int T, int U, int V1, uint32_t* __restrict__ bp, int* __restrict__ frames,
                                 float* __restrict__ token_logp, float* __restrict__ viterbi_logp, float* __restrict__ log_likelihood,
                                 int* __restrict__ path_rows) {
  extern __shared__ float4 smem_f4[];
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
  const int Tb = min(max(enc_len[b], 0), T), Ub = min(max(target_len[b], 0), U);
  const int S = 2 * Ub + 1, Smax = 2 * U + 1, W = (Smax + 15) / 16;
  int* lab_s = reinterpret_cast<int*>(smem_f4);   // [Smax]: l'_s | kSkip
  float* va = reinterpret_cast<float*>(lab_s + Smax);
  float* vb = va + Smax;
  float* fa = vb + Smax;
  float* fb = fa + Smax;
  __shared__ int final_s;
  const int blank = V1 - 1;
  const int* y = targets + static_cast<int64_t>(b) * U;
  int bad = 0;
  for (int s = tid; s < S; s += nt) {
    int l = blank;
    if (s & 1) {
      l = y[s >> 1];
      if (l < 0 || l >= blank) bad = 1;
      else if (s >= 3 && l != y[(s >> 1) - 1]) l |= kSkip;
    }
    lab_s[s] = l;
  }
  bad = __syncthreads_or(bad);
  const float* lp = log_probs + static_cast<int64_t>(b) * T * V1;
  uint32_t* bpu = bp + static_cast<int64_t>(b) * T * W;
  float vit = -INFINITY, fwd = -INFINITY;
  int nan = 0;
  if (!bad && Tb > 0) {
    for (int s = tid; s < S; s += nt) {
      const float x = s < 2 ? lp[lab_s[s] & ~kSkip] : -INFINITY;
      nan |= isnan(x);
      va[s] = fa[s] = x;
    }
    for (int s = tid; s < S; s += nt) {   // frame 0 reads every state's entry: the NaN rule counts them
      if (s >= 2) nan |= isnan(lp[lab_s[s] & ~kSkip]);
    }
    for (int t = 1; t < Tb; ++t) {
      __syncthreads();   // frame t - 1 complete
      const float* row = lp + static_cast<int64_t>(t) * V1;
      for (int s0 = 0; s0 < S; s0 += nt) {   // uniform trip count: whole warps take part in the shuffles
        const int s = s0 + tid;
        uint32_t code = 0;
        if (s < S) {
          const int l = lab_s[s];
          float best = va[s];
          float fm1 = -INFINITY, fm2 = -INFINITY;
          if (s >= 1) {
            const float c = va[s - 1];
            if (c > best) { best = c; code = 1; }
            fm1 = fa[s - 1];
          }
          if (l & kSkip) {
            const float c = va[s - 2];
            if (c > best) { best = c; code = 2; }
            fm2 = fa[s - 2];
          }
          const float x = row[l & ~kSkip];
          nan |= isnan(x);
          vb[s] = x + best;
          fb[s] = x + lse3(fa[s], fm1, fm2);
        }
        uint32_t word = code << (2 * (lane & 15));
#pragma unroll
        for (int off = 1; off < 16; off <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, off);
        if ((lane & 15) == 0 && s < S) bpu[static_cast<int64_t>(t) * W + s / 16] = word;
      }
      float* tmp = va; va = vb; vb = tmp;
      tmp = fa; fa = fb; fb = tmp;
    }
  }
  nan = __syncthreads_or(nan);   // also completes the last frame
  if (tid == 0) {
    int fs = -1;
    if (!bad && !nan && Tb > 0) {
      fs = S - 1;
      vit = va[S - 1];
      fwd = fa[S - 1];
      if (S >= 2) {
        if (va[S - 2] > vit) { vit = va[S - 2]; fs = S - 2; }
        fwd = lse2(fa[S - 1], fa[S - 2]);
      }
    }
    if (bad || nan) vit = fwd = qnan();
    viterbi_logp[b] = vit;
    log_likelihood[b] = fwd;
    path_rows[b] = Tb;
    final_s = (vit == -INFINITY || vit != vit) ? -1 : fs;
  }
  __syncthreads();
  int* fr = frames + static_cast<int64_t>(b) * U;
  float* tl = token_logp + static_cast<int64_t>(b) * U;
  const int fs = final_s;
  for (int i = tid; i < U; i += nt) fr[i] = -1;
  __syncthreads();
  if (fs >= 0 && tid == 0) {   // serial backtrack: a token's frame is the first frame of its run
    int s = fs;
    for (int t = Tb - 1; t >= 0; --t) {
      if (s & 1) fr[s >> 1] = t;
      if (t > 0) s -= (bpu[static_cast<int64_t>(t) * W + s / 16] >> (2 * (s & 15))) & 3u;
    }
  }
  __syncthreads();
  for (int i = tid; i < U; i += nt) {
    float v = -INFINITY;
    if (i < Ub) {
      if (bad || nan) v = qnan();
      else if (fs >= 0) v = lp[static_cast<int64_t>(fr[i]) * V1 + y[i]];
    }
    tl[i] = v;
  }
}

// blank / label [B, T, U + 1]; bp: B * (T + U) * W words, W = rnnt_bp_words(U)
__global__ void rnnt_align_kernel(const float* __restrict__ blank, const float* __restrict__ label, const int* __restrict__ enc_len,
                                  const int* __restrict__ target_len, int T, int U, uint32_t* __restrict__ bp, int* __restrict__ frames,
                                  float* __restrict__ token_logp, float* __restrict__ viterbi_logp, float* __restrict__ log_likelihood,
                                  int* __restrict__ path_rows) {
  extern __shared__ float4 smem_f4[];
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
  const int U1 = U + 1, W = (U1 + 31) / 32;
  const int Tb = min(max(enc_len[b], 0), T), Ub = min(max(target_len[b], 0), U);
  float* va = reinterpret_cast<float*>(smem_f4);   // [U1] per diagonal, indexed by u
  float* vb = va + U1;
  float* fa = vb + U1;
  float* fb = fa + U1;
  __shared__ int ok_s;
  const float* bl = blank + static_cast<int64_t>(b) * T * U1;
  const float* lb = label + static_cast<int64_t>(b) * T * U1;
  uint32_t* bpu = bp + static_cast<int64_t>(b) * (T + U) * W;
  int nan = 0;
  if (Tb > 0) {
    if (tid == 0) va[0] = fa[0] = 0.f;
    const int D = Tb - 1 + Ub;
    for (int d = 1; d <= D; ++d) {
      __syncthreads();   // diagonal d - 1 complete
      const int lo = max(0, d - (Tb - 1)), hi = min(Ub, d);
      for (int u0 = 0; u0 <= hi; u0 += nt) {   // uniform trip count for the ballot
        const int u = u0 + tid;
        bool take = false;
        if (u >= lo && u <= hi) {
          const int t = d - u;
          float cb = -INFINITY, cl = -INFINITY, fbk = -INFINITY, flk = -INFINITY;
          if (t > 0) {
            const float x = bl[static_cast<int64_t>(t - 1) * U1 + u];
            nan |= isnan(x);
            cb = va[u] + x;
            fbk = fa[u] + x;
          }
          if (u > 0) {
            const float x = lb[static_cast<int64_t>(t) * U1 + u - 1];
            nan |= isnan(x);
            cl = va[u - 1] + x;
            flk = fa[u - 1] + x;
            take = t == 0 || cl > cb;   // ties: the blank edge
          }
          vb[u] = take ? cl : cb;
          fb[u] = lse2(fbk, flk);
        }
        const uint32_t word = __ballot_sync(0xffffffffu, take);
        if (lane == 0 && u <= hi) bpu[static_cast<int64_t>(d) * W + u / 32] = word;
      }
      float* tmp = va; va = vb; vb = tmp;
      tmp = fa; fa = fb; fb = tmp;
    }
  }
  // the closing blank edge is read before the reduction, so that a NaN there reaches every thread's flag
  float x_end = 0.f;
  if (tid == 0 && Tb > 0) {
    x_end = bl[static_cast<int64_t>(Tb - 1) * U1 + Ub];
    nan |= isnan(x_end);
  }
  nan = __syncthreads_or(nan);
  if (tid == 0) {
    float vit = -INFINITY, fwd = -INFINITY;
    if (Tb > 0) {
      vit = va[Ub] + x_end;
      fwd = fa[Ub] + x_end;
    }
    if (nan) vit = fwd = qnan();
    viterbi_logp[b] = vit;
    log_likelihood[b] = fwd;
    path_rows[b] = Tb + Ub;
    ok_s = !(vit == -INFINITY || vit != vit);
  }
  __syncthreads();
  int* fr = frames + static_cast<int64_t>(b) * U;
  float* tl = token_logp + static_cast<int64_t>(b) * U;
  const int ok = ok_s;
  for (int i = tid; i < U; i += nt) fr[i] = -1;
  __syncthreads();
  if (ok && tid == 0) {   // serial backtrack from (Tb - 1, Ub): a label edge out of (t, u - 1) emits token u - 1 at frame t
    int t = Tb - 1, u = Ub;
    while (t + u > 0) {
      if ((bpu[static_cast<int64_t>(t + u) * W + u / 32] >> (u & 31)) & 1u) {
        fr[u - 1] = t;
        --u;
      } else {
        --t;
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < U; i += nt) {
    float v = -INFINITY;
    if (i < Ub) {
      if (nan) v = qnan();
      else if (ok) v = lb[static_cast<int64_t>(fr[i]) * U1 + i];
    }
    tl[i] = v;
  }
}

// ctc_align_kernel over a cluster of C = %cluster_nctarank CTAs per utterance (blockIdx.x / C); bp as there.  CTA k owns
// states [k P, min((k + 1) P, S)): 20 bytes of shared memory per state (label, two Viterbi and two forward buffers).
// Frame t reads frame t - 1's buffer, of this CTA and of CTA k - 1 (states s - 1 and s - 2 of the first two states), and
// writes the other buffer; one cluster barrier (release / acquire) per frame.  CTA k - 1 overwrites the buffer that CTA k
// reads in frame t only in frame t + 1, after the barrier that CTA k reaches when its frame t is done, so one barrier per
// frame is enough.  Every CTA checks all target ids itself, so `bad` needs no exchange; the NaN flags and the final states
// are read by CTA 0, which then backtracks (the last barrier makes every CTA's backpointer stores visible to it) and
// writes all outputs.
// GAPS: a boundary state (kBound) emits max(lp[t, blank], m[t] + log theta) in both recursions, every frame t < T_b also reads
// m[t] (a NaN there poisons the recording), and CTA 0's backtrack flags the unmatched frames; g is not read otherwise.
// SKIPS (with GAPS): the exit blank x_i of every line also takes the skip edge from (t - 1, e_i), compared after stay and
// s - 1, with backpointer code 3 (unused on blank states otherwise).  A blank's label is always blank, so its lab_s entry
// holds kSkip and the source instead: bits 16..19 its CTA j <= k, bits 0..15 its index there.  The source is read from frame
// t - 1's buffer, over distributed shared memory when j < k.  That is safe for the reason the left neighbour's read is: CTA
// j rewrites that buffer only in frame t + 1, after the barrier that CTA k reaches once its own frame t is done.  CTA 0's
// backtrack finds e_i again from line_edges (the other CTAs may have exited), leaves the jumped tokens at frame -1 and
// sums the penalties of the skip edges taken in frame order.
template <bool GAPS, bool SKIPS>
__global__ void ctc_align_long_kernel(const float* __restrict__ log_probs, const int* __restrict__ enc_len,
                                      const int* __restrict__ targets, const int* __restrict__ target_len, int T, int U, int V1, int P,
                                      uint32_t* __restrict__ bp, int* __restrict__ frames, float* __restrict__ token_logp,
                                      float* __restrict__ viterbi_logp, float* __restrict__ log_likelihood, int* __restrict__ path_rows,
                                      AlignGaps g) {
  static_assert(GAPS || !SKIPS, "skip mode runs on top of gap mode");
  constexpr int kLab = GAPS ? ~(kSkip | kBound) : ~kSkip;   // the label of a lab_s entry (odd states, in skip mode)
  extern __shared__ float4 smem_f4[];
  uint32_t C;
  asm("mov.u32 %0, %%cluster_nctarank;" : "=r"(C));
  const int k = static_cast<int>(ptx::cluster_ctarank());
  const int b = blockIdx.x / C, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
  const int Tb = min(max(enc_len[b], 0), T), Ub = min(max(target_len[b], 0), U);
  const int S = 2 * Ub + 1, Smax = 2 * U + 1, W = (Smax + 15) / 16;
  const int s0 = k * P, n = min(P, S - s0);   // this CTA's states of the utterance (none when n <= 0)
  int* lab_s = reinterpret_cast<int*>(smem_f4);   // [P]: l'_s | kSkip
  float* vbuf = reinterpret_cast<float*>(lab_s + P);   // [2][P]: frame t in buffer t & 1
  float* fbuf = vbuf + 2 * P;                          // [2][P]
  __shared__ int nan_s, poison_s, final_s;
  const int blank = V1 - 1;
  const int* y = targets + static_cast<int64_t>(b) * U;
  const uint8_t* edges = GAPS ? g.line_edges + static_cast<int64_t>(b) * U : nullptr;
  const float* mb = GAPS ? g.m + static_cast<int64_t>(b) * T : nullptr;
  int bad = 0;
  for (int i = tid; i < Ub; i += nt) {
    const int l = y[i];
    if (l < 0 || l >= blank) bad = 1;
  }
  for (int i = tid; i < n; i += nt) {
    const int s = s0 + i;
    int l = blank;
    if (s & 1) {
      l = y[s >> 1];
      if (l >= 0 && l < blank && s >= 3 && l != y[(s >> 1) - 1]) l |= kSkip;
    } else if (GAPS && boundary_state(edges, Ub, s)) {
      l |= kBound;
      if (SKIPS && s >= 2 && (edges[(s >> 1) - 1] & 2)) {   // x_i: keeps the source instead of the label
        const int e = skip_source(edges, s);
        l = kSkip | kBound | ((e / P) << kSrcIndexBits) | (e % P);
      }
    }
    lab_s[i] = l;
  }
  bad = __syncthreads_or(bad);
  const float* lp = log_probs + static_cast<int64_t>(b) * T * V1;
  uint32_t* bpu = bp + static_cast<int64_t>(b) * T * W;
  // frame buffers of CTA k - 1, as shared::cluster addresses
  const uint32_t left_v = k > 0 ? ptx::mapa_u32(ptx::smem_u32(vbuf), k - 1) : 0u;
  const uint32_t left_f = k > 0 ? ptx::mapa_u32(ptx::smem_u32(fbuf), k - 1) : 0u;
  int nan = 0;
  if (!bad && Tb > 0) {   // uniform over the cluster: every barrier below is reached by all of its threads
    float gt = 0.f;   // gap mode: m[t] + log theta of the current frame
    if constexpr (GAPS) {
      nan |= isnan(mb[0]);
      gt = mb[0] + g.log_theta;
    }
    for (int i = tid; i < n; i += nt) {
      const int s = s0 + i;
      float x = lp[SKIPS && !(s & 1) ? blank : lab_s[i] & kLab];   // frame 0 reads every state's entry: the NaN rule counts them
      nan |= isnan(x);
      if (GAPS && (lab_s[i] & kBound)) x = fmaxf(x, gt);
      vbuf[i] = fbuf[i] = s < 2 ? x : -INFINITY;
    }
    for (int t = 1; t < Tb; ++t) {
      float mt = 0.f;
      if constexpr (GAPS) mt = mb[t];   // loaded ahead of the barrier
      ptx::cluster_sync();   // frame t - 1 complete in every CTA of the cluster
      if constexpr (GAPS) {
        nan |= isnan(mt);
        gt = mt + g.log_theta;
      }
      const int p = (t - 1) & 1;
      const float* va = vbuf + p * P;
      const float* fa = fbuf + p * P;
      float* vb = vbuf + (p ^ 1) * P;
      float* fb = fbuf + (p ^ 1) * P;
      const uint32_t lv = left_v + 4u * static_cast<uint32_t>(p * P), lf = left_f + 4u * static_cast<uint32_t>(p * P);
      const float* row = lp + static_cast<int64_t>(t) * V1;
      for (int i0 = 0; i0 < P; i0 += nt) {   // uniform trip count: whole warps take part in the shuffles
        const int i = i0 + tid, s = s0 + i;
        uint32_t code = 0;
        if (i < n) {
          const int l = lab_s[i];
          float best = va[i];
          float fm1 = -INFINITY, fm2 = -INFINITY;
          if (s >= 1) {
            float c;
            if (i >= 1) {
              c = va[i - 1];
              fm1 = fa[i - 1];
            } else {
              c = ptx::ld_cluster_f32(lv + 4u * (P - 1));
              fm1 = ptx::ld_cluster_f32(lf + 4u * (P - 1));
            }
            if (c > best) { best = c; code = 1; }
          }
          if ((l & kSkip) && (!SKIPS || (s & 1))) {
            float c;
            if (i >= 2) {
              c = va[i - 2];
              fm2 = fa[i - 2];
            } else {
              c = ptx::ld_cluster_f32(lv + 4u * (P - 2 + i));
              fm2 = ptx::ld_cluster_f32(lf + 4u * (P - 2 + i));
            }
            if (c > best) { best = c; code = 2; }
          } else if (SKIPS && (l & kSkip)) {   // x_i: the skip edge from e_i, penalty fp32(n_i) * log psi
            const int j = (l >> kSrcIndexBits) & ((1 << kSrcCtaBits) - 1), e = l & ((1 << kSrcIndexBits) - 1);
            float c, fe;
            if (j == k) {
              c = va[e];
              fe = fa[e];
            } else {
              const uint32_t off = 4u * static_cast<uint32_t>(p * P + e);
              c = ptx::ld_cluster_f32(ptx::mapa_u32(ptx::smem_u32(vbuf), j) + off);
              fe = ptx::ld_cluster_f32(ptx::mapa_u32(ptx::smem_u32(fbuf), j) + off);
            }
            const float pen = __fmul_rn(static_cast<float>((s - (j * P + e)) >> 1), g.log_psi);   // rounded: no FMA
            c = c + pen;
            fm2 = fe + pen;
            if (c > best) { best = c; code = 3; }
          }
          float x = row[SKIPS && !(s & 1) ? blank : l & kLab];
          nan |= isnan(x);
          if (GAPS && (l & kBound)) x = fmaxf(x, gt);
          vb[i] = x + best;
          fb[i] = x + lse3(fa[i], fm1, fm2);
        }
        uint32_t word = code << (2 * (lane & 15));
#pragma unroll
        for (int off = 1; off < 16; off <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, off);
        if ((lane & 15) == 0 && i < n) bpu[static_cast<int64_t>(t) * W + s / 16] = word;
      }
    }
  }
  nan = __syncthreads_or(nan);
  if (tid == 0) nan_s = nan;
  ptx::cluster_sync();   // the last frame, every CTA's flag and backpointer stores are visible to the whole cluster
  if (k == 0 && tid == 0) {
    for (uint32_t r = 1; r < C; ++r) nan |= ptx::ld_cluster_s32(ptx::mapa_u32(ptx::smem_u32(&nan_s), r));
    int fs = -1;
    float vit = -INFINITY, fwd = -INFINITY;
    if (!bad && !nan && Tb > 0) {
      const int p = (Tb - 1) & 1;
      auto at = [&](const float* buf, int s) {   // state s of the last frame, in whichever CTA owns it
        return ptx::ld_cluster_f32(ptx::mapa_u32(ptx::smem_u32(buf + p * P + s % P), s / P));
      };
      fs = S - 1;
      vit = at(vbuf, S - 1);
      fwd = at(fbuf, S - 1);
      if (S >= 2) {
        const float v2 = at(vbuf, S - 2);
        if (v2 > vit) { vit = v2; fs = S - 2; }
        fwd = lse2(fwd, at(fbuf, S - 2));
      }
    }
    if (bad || nan) vit = fwd = qnan();
    viterbi_logp[b] = vit;
    log_likelihood[b] = fwd;
    path_rows[b] = Tb;
    poison_s = bad || nan;
    final_s = (vit == -INFINITY || vit != vit) ? -1 : fs;
  }
  ptx::cluster_sync();   // CTA 0 is done reading the others' shared memory: they may exit
  if (k != 0) return;
  int* fr = frames + static_cast<int64_t>(b) * U;
  float* tl = token_logp + static_cast<int64_t>(b) * U;
  const int fs = final_s, poison = poison_s;
  uint8_t* um = GAPS ? g.unmatched + static_cast<int64_t>(b) * T : nullptr;
  for (int i = tid; i < U; i += nt) fr[i] = -1;
  if constexpr (GAPS)
    for (int t = tid; t < T; t += nt) um[t] = 0;
  __syncthreads();
  if (fs >= 0 && tid == 0) {   // serial backtrack, as ctc_align_kernel's
    int s = fs, rows = 0, skips = 0;
    for (int t = Tb - 1; t >= 0; --t) {
      if (s & 1) {
        fr[s >> 1] = t;
      } else if (GAPS && boundary_state(edges, Ub, s) && mb[t] + g.log_theta > lp[static_cast<int64_t>(t) * V1 + blank]) {
        um[t] = 1;   // the sweep's boundary emission took m[t] + log theta here
        ++rows;
      }
      if (t > 0) {
        const uint32_t code = (bpu[static_cast<int64_t>(t) * W + s / 16] >> (2 * (s & 15))) & 3u;
        if (SKIPS && code == 3) {   // the tokens of (e_i, x_i) keep frame -1
          s = skip_source(edges, s);
          ++skips;
        } else {
          s -= code;
        }
      }
    }
    if constexpr (GAPS) {
      float sum = 0.f;
      for (int t = 0; t < Tb; ++t)
        if (um[t]) sum += mb[t] + g.log_theta;   // in frame order
      g.unmatched_rows[b] = rows;
      g.unmatched_logp[b] = sum;
    }
    if constexpr (SKIPS) {   // skip edge i is on the path iff line i's last token was jumped; frame order is line order
      float sum = 0.f;
      for (int j = 0, e = 0; skips > 0 && j < Ub; ++j) {
        if (edges[j] & 2) {
          if (fr[j] < 0) sum += __fmul_rn(static_cast<float>(j + 1 - e / 2), g.log_psi);
          e = 2 * (j + 1);
        }
      }
      g.skipped_rows[b] = skips;
      g.skip_logp[b] = sum;
    }
  }
  if (GAPS && tid == 0 && fs < 0) {   // no path, or poisoned
    g.unmatched_rows[b] = 0;
    g.unmatched_logp[b] = poison ? qnan() : 0.f;
    if constexpr (SKIPS) {
      g.skipped_rows[b] = 0;
      g.skip_logp[b] = poison ? qnan() : 0.f;
    }
  }
  __syncthreads();
  for (int i = tid; i < U; i += nt) {
    float v = -INFINITY;
    if (i < Ub) {
      if (poison) v = qnan();
      else if (fs >= 0 && (!SKIPS || fr[i] >= 0)) v = lp[static_cast<int64_t>(fr[i]) * V1 + y[i]];
    }
    tl[i] = v;
  }
}

// gap mode's pre-pass: m[b, t] = max_c lp[t, c] (warp_row_max) for t < T_b, one warp per frame, strided over t and b
__global__ void row_max_kernel(const float* __restrict__ log_probs, const int* __restrict__ enc_len, int B, int T, int V1,
                               float* __restrict__ m) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const int Tb = min(max(enc_len[b], 0), T);
    for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < Tb; t += gridDim.x * wpb) {   // whole warps
      const int64_t r = static_cast<int64_t>(b) * T + t;
      const float mx = warp_row_max(log_probs + r * V1, V1, lane);
      if (lane == 0) m[r] = mx;
    }
  }
}

// cluster and shared-memory attributes of one instantiation, once per device
template <bool GAPS, bool SKIPS>
int align_long_attributes() {
  static PerDeviceOnce attr_once;
  if (!attr_once.first()) return 0;
  int dev = 0, cap = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (cudaFuncSetAttribute(ctc_align_long_kernel<GAPS, SKIPS>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
      cudaFuncSetAttribute(ctc_align_long_kernel<GAPS, SKIPS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           cap - kAlignLongStaticSmem) != cudaSuccess)
    return -1;
  return 0;
}

int align_threads(int n) { return n <= 64 ? 64 : n >= 1024 ? 1024 : (n + 31) / 32 * 32; }

}  // namespace

int64_t ctc_bp_words(int T, int U) { return static_cast<int64_t>(T) * ((2 * U + 1 + 15) / 16); }
int64_t rnnt_bp_words(int T, int U) { return static_cast<int64_t>(T + U) * ((U + 1 + 31) / 32); }

int launch_ctc_align(const float* log_probs, const int* enc_len, const int* targets, const int* target_len, int B, int T, int U, int V1,
                     uint32_t* bp, int* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int* path_rows,
                     cudaStream_t s) {
  static PerDeviceOnce attr_once;
  if (U > kAlignMaxTokens) return 1;
  if (attr_once.first() && cudaFuncSetAttribute(ctc_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                5 * (2 * kAlignMaxTokens + 1) * 4) != cudaSuccess)
    return -1;
  const size_t smem = static_cast<size_t>(5) * (2 * U + 1) * 4;
  ctc_align_kernel<<<B, align_threads(2 * U + 1), smem, s>>>(log_probs, enc_len, targets, target_len, T, U, V1, bp, frames, token_logp,
                                                            viterbi_logp, log_likelihood, path_rows);
  return 0;
}

int ctc_align_long_plan(int U, int forced_ctas, int* ctas, int* states_per_cta) {
  if (U < 0 || U > kAlignLongMaxTokens || forced_ctas < 0 || forced_ctas > kAlignLongMaxCtas) return 1;
  int dev = 0, cap = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return -1;
  const int smax = 2 * U + 1;
  const int lo = forced_ctas ? forced_ctas : 1, hi = forced_ctas ? forced_ctas : kAlignLongMaxCtas;
  for (int c = lo; c <= hi; ++c) {
    const int p = ((smax + c - 1) / c + 15) / 16 * 16;
    if ((c - 1) * p >= smax) {   // CTA c - 1 would own no state
      if (forced_ctas) return 2;
      continue;
    }
    if (static_cast<int64_t>(p) * 20 + kAlignLongStaticSmem <= cap) {
      *ctas = c;
      *states_per_cta = p;
      return 0;
    }
  }
  return 1;
}

int launch_ctc_align_long(const float* log_probs, const int* enc_len, const int* targets, const int* target_len, int B, int T, int U,
                          int V1, int forced_ctas, uint32_t* bp, int* frames, float* token_logp, float* viterbi_logp,
                          float* log_likelihood, int* path_rows, int* plan, const AlignGaps* gaps, cudaStream_t s) {
  int C = 0, P = 0;
  const int rc = ctc_align_long_plan(U, forced_ctas, &C, &P);
  if (rc != 0) return rc;
  const bool skips = gaps && gaps->skipped_rows;
  if (skips && P > (1 << kSrcIndexBits)) return 1;   // a source index would not fit in its lab_s field
  if ((skips  ? align_long_attributes<true, true>()
       : gaps ? align_long_attributes<true, false>()
              : align_long_attributes<false, false>()) != 0)
    return -1;
  if (plan) {
    plan[0] = C;
    plan[1] = P;
  }
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = C;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(static_cast<unsigned>(B) * C);
  cfg.blockDim = dim3(align_threads(P));
  cfg.dynamicSmemBytes = static_cast<size_t>(P) * 20;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (!gaps)
    return cudaLaunchKernelEx(&cfg, ctc_align_long_kernel<false, false>, log_probs, enc_len, targets, target_len, T, U, V1, P, bp, frames,
                              token_logp, viterbi_logp, log_likelihood, path_rows, AlignGaps{}) != cudaSuccess
               ? -2
               : 0;
  const dim3 grid(static_cast<unsigned>(std::min<int64_t>((static_cast<int64_t>(T) + 7) / 8, 65535)), std::min(B, 65535));
  row_max_kernel<<<grid, 256, 0, s>>>(log_probs, enc_len, B, T, V1, gaps->m);
  if (cudaLaunchKernelEx(&cfg, skips ? ctc_align_long_kernel<true, true> : ctc_align_long_kernel<true, false>, log_probs, enc_len, targets, target_len, T, U, V1, P, bp, frames, token_logp,
                         viterbi_logp, log_likelihood, path_rows, *gaps) != cudaSuccess)
    return -2;
  return 0;
}

int launch_rnnt_align(const float* blank, const float* label, const int* enc_len, const int* target_len, int B, int T, int U, uint32_t* bp,
                      int* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int* path_rows, cudaStream_t s) {
  static PerDeviceOnce attr_once;
  if (U > kAlignMaxTokens) return 1;
  if (attr_once.first() && cudaFuncSetAttribute(rnnt_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                4 * (kAlignMaxTokens + 1) * 4) != cudaSuccess)
    return -1;
  const size_t smem = static_cast<size_t>(4) * (U + 1) * 4;
  rnnt_align_kernel<<<B, align_threads(U + 1), smem, s>>>(blank, label, enc_len, target_len, T, U, bp, frames, token_logp, viterbi_logp,
                                                          log_likelihood, path_rows);
  return 0;
}

}  // namespace gam
