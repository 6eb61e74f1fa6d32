// GigaAMEmo over time.  The head is Linear(768, C) on the mean of the encoder frames, so in real arithmetic
// softmax(W mean_t f_t + b) = softmax(mean_t (W f_t + b)): the emotion of any span of frames follows from the per-frame
// logits l_t = W f_t + b alone, C numbers per frame.  fp32 on the CUDA cores, like pooled_head.cu.
//   (1) emo_frame_logits_kernel: row b's local frames t in [lo', hi') of enc [B, T, 768] (lo[b], hi[b] clamped to [0, T])
//       -> frame_logits rows dst[b] + t - lo'.  A warp takes one frame at a time (lane l holds k = 4l + 128 i, i < 6, in
//       registers) and runs pooled_head_kernel's dot product for every class: lane l sums its k in ascending i with fmaf,
//       then the same xor tree, then + bias.  A frame's logits thus have the same bits whichever row, window or launch produced them.  W and
//       b are staged in shared memory when they fit in the default 48 KiB of a CTA (C <= 15), else read through L1 / L2.
//   (2) emo_spans_kernel: one CTA per span [a, b) of frame_logits -> the mean of l over the span (pool_chunks_kernel's
//       order: kPoolChunk-frame sums in ascending t, then the chunk sums from 0 in ascending order, then / n) and its
//       softmax (pooled_head_kernel's block max, expf and block sum).  The order depends on the span's length only.
// No atomics, no allocation, no host synchronisation: both launches can be captured in a CUDA graph.
#include <cmath>

#include "kernels.h"

namespace gam {
namespace {

constexpr int kD = 768;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kFramesPerCta = 64;               // (1): local frames per CTA, kFramesPerCta / kWarps per warp
constexpr int kSmemBudget = 48 * 1024;          // (1): W and b staged only within the default dynamic shared memory
static_assert(kThreads == kPoolMaxClasses, "the softmax keeps one class per thread");

__host__ __device__ constexpr int staged_bytes(int C) { return (C * kD + ((C + 3) & ~3)) * 4; }

template <bool kStaged>
__global__ void __launch_bounds__(kThreads) emo_frame_logits_kernel(const float* __restrict__ enc, int T, const int* __restrict__ lo_v,
                                                                   const int* __restrict__ hi_v, const int* __restrict__ dst_v,
                                                                   const float* __restrict__ W, const float* __restrict__ bias, int C,
                                                                   float* __restrict__ out, int n_frames) {
  extern __shared__ __align__(16) float w_s[];
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lo = min(max(lo_v[b], 0), T), hi = min(max(hi_v[b], 0), T);
  const int t0 = lo + blockIdx.x * kFramesPerCta;
  if (t0 >= hi) return;                          // the same test for every thread: no barrier is skipped by some only
  const int t1 = min(t0 + kFramesPerCta, hi);
  const int64_t shift = static_cast<int64_t>(dst_v[b]) - lo;
  const float* Wp = W;
  const float* bp = bias;
  if constexpr (kStaged) {
    const float4* src = reinterpret_cast<const float4*>(W);
    float4* w4 = reinterpret_cast<float4*>(w_s);
    for (int i = threadIdx.x; i < C * kD / 4; i += kThreads) w4[i] = __ldg(src + i);
    float* b_s = w_s + C * kD;
    for (int i = threadIdx.x; i < C; i += kThreads) b_s[i] = __ldg(bias + i);
    __syncthreads();
    Wp = w_s;
    bp = b_s;
  }
  for (int t = t0 + warp; t < t1; t += kWarps) {
    const int64_t row = t + shift;
    if (row < 0 || row >= n_frames) continue;    // writes outside [0, n_frames) are dropped
    const float4* f4 = reinterpret_cast<const float4*>(enc + (static_cast<int64_t>(b) * T + t) * kD);
    float4 f[kD / 128];
#pragma unroll
    for (int i = 0; i < kD / 128; ++i) f[i] = __ldg(f4 + lane + 32 * i);
    float* o = out + row * C;
    float mine = 0.f;
    for (int c = 0; c < C; ++c) {
      const float4* w4 = reinterpret_cast<const float4*>(Wp + static_cast<int64_t>(c) * kD);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < kD / 128; ++i) {
        const float4 w = kStaged ? w4[lane + 32 * i] : __ldg(w4 + lane + 32 * i);
        acc = fmaf(w.x, f[i].x, acc);
        acc = fmaf(w.y, f[i].y, acc);
        acc = fmaf(w.z, f[i].z, acc);
        acc = fmaf(w.w, f[i].w, acc);
      }
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      // every lane holds the same sum; lane c % 32 keeps class c and each run of 32 classes is stored at once
      if (lane == (c & 31)) mine = acc + (kStaged ? bp[c] : __ldg(bp + c));
      if ((c & 31) == 31 || c == C - 1) {
        if (lane <= (c & 31)) o[(c & ~31) + lane] = mine;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) emo_spans_kernel(const float* __restrict__ fl, int n_frames, int C,
                                                            const int* __restrict__ span_start, const int* __restrict__ span_end,
                                                            float* __restrict__ logits, float* __restrict__ probs) {
  __shared__ float part_s[kThreads];
  __shared__ float red_s[kWarps];
  const int sp = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a = min(max(span_start[sp], 0), n_frames);
  const int n = max(min(max(span_end[sp], 0), n_frames) - a, 0);
  const int nc = (n + kPoolChunk - 1) / kPoolChunk;
  // chunk sums of G chunks at a time, G C <= 256 threads: thread (j, c) sums chunk g + j of class c in ascending t from its
  // first frame, then thread c adds the G sums to its running total in ascending chunk order
  const int G = max(1, kThreads / C);
  const int j = tid / C, cj = tid - j * C;
  const bool worker = j < G;
  float total = 0.f;
  for (int g = 0; g < nc; g += G) {
    if (worker && g + j < nc) {
      const int f0 = a + (g + j) * kPoolChunk, f1 = min(f0 + kPoolChunk, a + n);
      const float* p = fl + static_cast<int64_t>(f0) * C + cj;
      float s = p[0];
      for (int t = f0 + 1; t < f1; ++t) s += p[static_cast<int64_t>(t - f0) * C];
      part_s[tid] = s;
    }
    __syncthreads();
    if (tid < C) {
      const int m = min(G, nc - g);
      for (int q = 0; q < m; ++q) total += part_s[q * C + tid];
    }
    __syncthreads();
  }
  const bool live = tid < C;
  const float v = live ? total / static_cast<float>(n) : -INFINITY;   // n == 0: 0 / 0 = NaN, the mean of an empty set
  if (live && logits != nullptr) logits[static_cast<int64_t>(sp) * C + tid] = v;
  if (probs == nullptr) return;
  // softmax exactly as pooled_head_kernel: block max, exp, block sum (xor tree in each warp, then the warp partials in order)
  float m = v;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if (lane == 0) red_s[warp] = m;
  __syncthreads();
  m = red_s[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) m = fmaxf(m, red_s[w]);
  __syncthreads();
  float e = live ? expf(v - m) : 0.f;
  float s = e;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) red_s[warp] = s;
  __syncthreads();
  s = red_s[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) s += red_s[w];
  if (live) probs[static_cast<int64_t>(sp) * C + tid] = e / s;
}

}  // namespace

void launch_emo_frame_logits(const float* enc, int B, int T, const int* lo, const int* hi, const int* dst, const float* W,
                             const float* bias, int C, float* frame_logits, int n_frames, cudaStream_t s) {
  const dim3 grid((T + kFramesPerCta - 1) / kFramesPerCta, B);
  const int smem = staged_bytes(C);
  if (smem <= kSmemBudget)
    emo_frame_logits_kernel<true><<<grid, kThreads, smem, s>>>(enc, T, lo, hi, dst, W, bias, C, frame_logits, n_frames);
  else
    emo_frame_logits_kernel<false><<<grid, kThreads, 0, s>>>(enc, T, lo, hi, dst, W, bias, C, frame_logits, n_frames);
}

void launch_emo_spans(const float* frame_logits, int n_frames, int C, const int* span_start, const int* span_end, int S, float* logits,
                      float* probs, cudaStream_t s) {
  emo_spans_kernel<<<S, kThreads, 0, s>>>(frame_logits, n_frames, C, span_start, span_end, logits, probs);
}

}  // namespace gam
