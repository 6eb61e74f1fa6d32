// CTC head + greedy decode (gigaam/decoder.py:7-21, gigaam/decoding.py:56-96).
//   (1) head + argmax: labels[b,t] = argmax_c (W[c,:] . enc[b,t,:] + bias[c]) in fp32 - log_softmax is
//       argmax-invariant on finite rows so it is never computed.  The label is torch's log_softmax(row).argmax(-1):
//       on a row whose maximum is finite the first maximal index (torch.argmax); if any logit is NaN or +inf, or none
//       exceeds -inf, 0 (log_softmax makes such a row all NaN).  Always in [0, V1).
//   (2) collapse: keep (l != blank) && (l != l_{t-1}) && (t < len); one warp per utterance, ballot + popc prefix
//       compaction, results resident on device: ids, frames, counts (int32).  One kernel serves the one-shot calls (a
//       fresh stream) and gam_ctc_greedy_resume (a stream continued from its DecodeState).
//   Scored (gam_ctc_greedy_scored, scored resume): the argmax also keeps, per class group, the running sum of exp(z_c - best)
//   beside its (best value, index), rescaled whenever the best moves; the groups merge in the same shared-memory merge and
//   the frame's l = log_softmax(row)[label] = -log sum_c exp(z_c - z_max) goes to scratch (NaN on a row whose label is
//   0 by the non-finite rule).  The logits are the same fp32 sums in the same k order, so the labels are the unscored
//   kernel's.  The scored collapse gathers l at the emitted frames and sums it over t < len in fp64, in an order fixed by
//   t alone (lane-strided partial sums, then a fixed xor tree), so an utterance's scores do not depend on its batch.
#include "kernels.h"

namespace gam {
namespace {

constexpr int kRows = 32;      // rows (frames) per block: thread = (row, class group)
constexpr int kGroups = 4;     // class groups = warps per block
constexpr int kKC = 64;        // K chunk
constexpr int kCG = 9;         // classes per thread and class tile
constexpr int kCT = kGroups * kCG;   // class tile (36)

// enc: [R, D] fp32 row-major.  W: [V1, D], bias [V1].  labels: [R] int32.
// Block = 32 frames x 4 class groups (one warp per group: its W reads are broadcasts, its enc reads conflict-free):
// 502 blocks at the benchmark shape instead of 126 single-warp-per-SM blocks.
// Every (frame, class) sum still runs over k in ascending order, so the logits -- and the argmax -- are bit-identical.
// SCORED: also lp[R] = l of every row (the unscored instantiation computes and stores nothing more).
template <bool SCORED>
__global__ void __launch_bounds__(kRows * kGroups) ctc_argmax_kernel(const float* __restrict__ enc, const float* __restrict__ W,
                                                                     const float* __restrict__ bias, int* __restrict__ labels,
                                                                     int R, int D, int V1, float* __restrict__ lp) {
  __shared__ float e_s[kKC][kRows + 1];
  __shared__ float w_s[kCT][kKC];
  __shared__ float best_v[kGroups][kRows];
  __shared__ int best_c[kGroups][kRows];
  __shared__ float best_s[SCORED ? kGroups : 1][kRows];
  const int r = threadIdx.x & 31, cg = threadIdx.x >> 5;
  const int row0 = blockIdx.x * kRows;
  float best = -INFINITY;
  int best_i = 0;
  [[maybe_unused]] float sum = 0.f;   // SCORED: sum of exp(v - best) over this group's finite logits so far
  for (int c0 = 0; c0 < V1; c0 += kCT) {
    float acc[kCG];
#pragma unroll
    for (int c = 0; c < kCG; ++c) acc[c] = 0.f;
    for (int k0 = 0; k0 < D; k0 += kKC) {
      __syncthreads();
      // enc tile: coalesced float4 reads along K, transposed into e_s[k][row]
      for (int i = threadIdx.x; i < kRows * (kKC / 4); i += kRows * kGroups) {
        const int rr = i / (kKC / 4), k4 = (i % (kKC / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row0 + rr < R) v = *reinterpret_cast<const float4*>(enc + static_cast<size_t>(row0 + rr) * D + k0 + k4);
        e_s[k4 + 0][rr] = v.x;
        e_s[k4 + 1][rr] = v.y;
        e_s[k4 + 2][rr] = v.z;
        e_s[k4 + 3][rr] = v.w;
      }
      for (int i = threadIdx.x; i < kCT * kKC; i += kRows * kGroups) {
        const int c = i / kKC, k = i % kKC;
        w_s[c][k] = (c0 + c < V1) ? __ldg(W + static_cast<size_t>(c0 + c) * D + k0 + k) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < kKC; ++k) {
        const float x = e_s[k][r];
#pragma unroll
        for (int c = 0; c < kCG; ++c) acc[c] = fmaf(w_s[cg * kCG + c][k], x, acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < kCG; ++c) {
      const int cls = c0 + cg * kCG + c;
      if (cls < V1) {
        const float v = acc[c] + __ldg(bias + cls);
        // ascending classes, strict >: first maximal index wins; a NaN or +inf logit becomes (+inf, -1), the
        // "non-finite seen" mark that no later logit replaces and that wins the merge below
        if (!(v <= best)) {
          const bool bad = !(v < INFINITY);
          if constexpr (SCORED) {
            if (!bad) sum = sum * expf(best - v) + 1.f;   // best = -inf at the start: 0 * 0 + 1
          }
          best = bad ? INFINITY : v;
          best_i = bad ? -1 : cls;
        } else if constexpr (SCORED) {
          if (v > -INFINITY) sum += expf(v - best);
        }
      }
    }
  }
  // merge the class groups; a group only ever holds classes c0 + cg * 9 + j, so "first maximal index" = smallest index
  // among equal values, decided explicitly
  best_v[cg][r] = best;
  best_c[cg][r] = best_i;
  if constexpr (SCORED) best_s[cg][r] = sum;
  __syncthreads();
  if (cg == 0 && row0 + r < R) {
#pragma unroll
    for (int g = 1; g < kGroups; ++g) {
      const float v = best_v[g][r];
      const int i = best_c[g][r];
      if (v > best || (v == best && i < best_i)) { best = v; best_i = i; }
    }
    labels[row0 + r] = best_i < 0 ? 0 : best_i;   // NaN or +inf in any group -> 0
    if constexpr (SCORED) {
      // the row's maximum is `best` whatever the merge order; the groups' sums are rescaled to it in group order.  A
      // row with a NaN / +inf logit (best_i < 0) or with no logit above -inf has l = NaN, as torch's log_softmax gives.
      float l = __int_as_float(0x7fffffff);
      if (best_i >= 0 && best > -INFINITY) {
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < kGroups; ++g) {
          const float v = best_v[g][r];
          if (v > -INFINITY) s += best_s[g][r] * expf(v - best);
        }
        l = -logf(s);
      }
      lp[row0 + r] = l;
    }
  }
}

// Greedy collapse of one utterance per warp (GreedyIo): keep (l != blank) && (l != prev) over frames [a, e), ballot + popc
// prefix compaction, appending at pos0.  A fresh call starts at a = 0 with prev = blank, pos0 = 0 and zero partials; a resume
// call takes prev, the rows so far and the partials from the stream's DecodeState.  The fresh rule keeps the tokens of the
// one-frame-back rule (t == 0 || l != l_{t-1}): at t = 0 a kept label is not the blank, so it differs from prev = blank.
// SCORED: token_logp = lp of the kept frame, and the path sum is taken in fp64 in an order fixed by the stream's row index
// r alone -- row r goes to lane partial r % 32 in ascending r (rot = 0 on a fresh call), and the 32 partials meet in one xor
// tree -- so decoding [0, L) in consecutive calls gives a fresh call's bits and scores do not depend on the batch.
template <bool SCORED>
__global__ void __launch_bounds__(128) ctc_collapse_kernel(const int* __restrict__ labels, const float* __restrict__ lp, int B, int T,
                                                           int blank, const GreedyIo io) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (b >= B) return;
  DecodeState* st = io.state ? reinterpret_cast<DecodeState*>(io.state + b * io.stride) : nullptr;
  const int a = st ? min(max(io.lo[b], 0), T) : 0, e = min(max(io.hi[b], a), T);
  if (st && a == e) return;   // a resume call leaves a stream without frames as it is
  const int* lab = labels + static_cast<size_t>(b) * T;
  const int fb = st ? io.frame_base[b] : 0, prev0 = st ? st->label : blank, rows0 = st ? st->rows : 0;
  const int pos0 = st ? io.counts[b] : 0;
  int pos = pos0;
  [[maybe_unused]] double part = 0.0;
  [[maybe_unused]] const int rot = rows0 & 31;   // lane k keeps partial k; row t comes from lane (k - rot) mod 32
  if constexpr (SCORED) {
    if (st) part = st->part[lane];
  }
  for (int t0 = a; t0 < e; t0 += 32) {
    const int t = t0 + lane;
    int l = blank, prev = blank;
    if (t < e) {
      l = lab[t];
      prev = t > a ? lab[t - 1] : prev0;
    }
    const bool keep = (t < e) && (l != blank) && (l != prev);
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    const int p = pos + __popc(mask & ((1u << lane) - 1u));
    [[maybe_unused]] float x = 0.f;
    if constexpr (SCORED) {
      if (t < e) {
        x = lp[static_cast<size_t>(b) * T + t];
        if (io.frame_logp) {
          io.frame_logp[b * io.frame_pitch + fb + t] = static_cast<double>(x);
          io.frame_rows[b * io.frame_pitch + fb + t] = 1;
        }
      }
    }
    if (keep && p < io.max_out) {
      io.ids[static_cast<size_t>(b) * io.max_out + p] = l;
      io.frames[static_cast<size_t>(b) * io.max_out + p] = fb + t;
      if constexpr (SCORED) io.token_logp[static_cast<size_t>(b) * io.max_out + p] = x;
    }
    if constexpr (SCORED) {
      const int src = (lane - rot) & 31;
      const float xs = __shfl_sync(0xffffffffu, x, src);
      if (t0 + src < e) part += static_cast<double>(xs);
    }
    pos += __popc(mask);
  }
  if constexpr (SCORED) {
    if (st) st->part[lane] = part;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  }
  if (lane == 0) {
    io.counts[b] = min(pos, io.max_out);
    if (st) {
      st->label = lab[e - 1];
      st->count += pos - pos0;
      if constexpr (SCORED) st->rows = rows0 + (e - a);
    }
    if constexpr (SCORED) {
      io.path_logp[b] = static_cast<float>(part);
      io.path_rows[b] = rows0 + (e - a);
    }
  }
}

__global__ void decode_state_init_kernel(uint8_t* state, int64_t stride, int n, int blank) {
  const int b = blockIdx.x;
  if (b >= n) return;
  uint32_t* w = reinterpret_cast<uint32_t*>(state + b * stride);
  for (int i = threadIdx.x; i < static_cast<int>(stride / 4); i += blockDim.x) w[i] = 0u;
  __syncthreads();
  if (threadIdx.x == 0) {
    DecodeState* st = reinterpret_cast<DecodeState*>(state + b * stride);
    st->label = blank;
    st->pending = 1;
  }
}

}  // namespace

void launch_decode_state_init(uint8_t* state, int64_t stride, int n, int blank, cudaStream_t s) {
  if (n > 0) decode_state_init_kernel<<<n, 256, 0, s>>>(state, stride, n, blank);
}
void launch_ctc_argmax(const float* enc, const float* W, const float* bias, int* labels, float* lp, int R, int D, int V1,
                       cudaStream_t s) {
  if (lp)
    ctc_argmax_kernel<true><<<(R + kRows - 1) / kRows, kRows * kGroups, 0, s>>>(enc, W, bias, labels, R, D, V1, lp);
  else
    ctc_argmax_kernel<false><<<(R + kRows - 1) / kRows, kRows * kGroups, 0, s>>>(enc, W, bias, labels, R, D, V1, nullptr);
}
void launch_ctc_collapse(const int* labels, const float* lp, int B, int T, int blank, const GreedyIo& io, cudaStream_t s) {
  if (io.token_logp)
    ctc_collapse_kernel<true><<<(B + 3) / 4, 128, 0, s>>>(labels, lp, B, T, blank, io);
  else
    ctc_collapse_kernel<false><<<(B + 3) / 4, 128, 0, s>>>(labels, lp, B, T, blank, io);
}

}  // namespace gam
