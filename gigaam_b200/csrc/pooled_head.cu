// Pooled classification head of GigaAMEmo (gigaam/model.py:272-293): the mean of the encoder output over an utterance's
// frames, a Linear(d, C) layer and a softmax over the C classes.  All arithmetic is fp32 on the CUDA cores, like the
// reference's fp32 head; the exponential is expf, as in heads.cu.
//   (1) pool_chunks_kernel: one CTA per (utterance, chunk of kPoolChunk frames) sums the chunk's frames in ascending t
//       into the workspace, four columns per thread.  Chunks at or past the utterance's length exit at once, so frames
//       t >= n_b are never read.
//   (2) pooled_head_kernel: one CTA per utterance adds its chunk sums in ascending chunk order, divides by n_b, then
//       computes logits = W pooled + b (a warp per class, lanes over k, a fixed xor-shuffle tree) and the softmax (a
//       thread per class).
// The summation order of utterance b depends only on n_b: neither B, T nor the neighbours change a bit of its result, and
// no float atomics are used.  Launches only (no allocation, no host synchronisation): the call can be captured in a
// CUDA graph.
#include <cmath>

#include "kernels.h"

namespace gam {
namespace {

constexpr int kPoolD = 768;                 // d_model the kernels are specialised for (gam_create refuses others)
constexpr int kPoolThreads = kPoolD / 4;    // (1): one float4 column group per thread
constexpr int kHeadThreads = 256;           // (2): one thread per class, C <= 256
constexpr int kHeadWarps = kHeadThreads / 32;
constexpr int kUnroll = 8;                  // (1): loads issued ahead of their adds
static_assert(kHeadThreads == kPoolMaxClasses, "the softmax keeps one class per thread");

// frames pooled for utterance b (the pack plan's plen rule): enc_len[b] clamped to [0, T], or all T frames for a batch
// of one or without lengths
__device__ __forceinline__ int pooled_frames(const int* __restrict__ enc_len, int B, int T, int b) {
  if (enc_len == nullptr || B == 1) return T;
  return min(max(enc_len[b], 0), T);
}

__global__ void __launch_bounds__(kPoolThreads) pool_chunks_kernel(const float* __restrict__ enc, const int* __restrict__ enc_len,
                                                                   int B, int T, int n_chunks, float* __restrict__ part) {
  const int b = blockIdx.x, chunk = blockIdx.y;
  const int n = pooled_frames(enc_len, B, T, b);
  const int t0 = chunk * kPoolChunk;
  if (t0 >= n) return;
  const int t1 = min(t0 + kPoolChunk, n);
  const float4* src = reinterpret_cast<const float4*>(enc + (static_cast<int64_t>(b) * T + t0) * kPoolD) + threadIdx.x;
  constexpr int kRow4 = kPoolD / 4;
  float4 s = src[0];
  int t = t0 + 1;
  for (; t + kUnroll <= t1; t += kUnroll) {
    float4 v[kUnroll];
#pragma unroll
    for (int i = 0; i < kUnroll; ++i) v[i] = src[static_cast<int64_t>(t - t0 + i) * kRow4];
#pragma unroll
    for (int i = 0; i < kUnroll; ++i) {
      s.x += v[i].x;
      s.y += v[i].y;
      s.z += v[i].z;
      s.w += v[i].w;
    }
  }
  for (; t < t1; ++t) {
    const float4 v = src[static_cast<int64_t>(t - t0) * kRow4];
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  reinterpret_cast<float4*>(part + (static_cast<int64_t>(b) * n_chunks + chunk) * kPoolD)[threadIdx.x] = s;
}

__global__ void __launch_bounds__(kHeadThreads) pooled_head_kernel(const float* __restrict__ part, const int* __restrict__ enc_len,
                                                                   int B, int T, int n_chunks, const float* __restrict__ W,
                                                                   const float* __restrict__ bias, int C,
                                                                   float* __restrict__ pooled, float* __restrict__ logits,
                                                                   float* __restrict__ probs) {
  __shared__ __align__(16) float p_s[kPoolD];
  __shared__ float l_s[kHeadThreads];
  __shared__ float red_s[kHeadWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = pooled_frames(enc_len, B, T, b);
  const int nc = (n + kPoolChunk - 1) / kPoolChunk;
  const float* pb = part + static_cast<int64_t>(b) * n_chunks * kPoolD;
  for (int col = tid; col < kPoolD; col += kHeadThreads) {
    float s = 0.f;
    for (int c = 0; c < nc; ++c) s += pb[static_cast<int64_t>(c) * kPoolD + col];
    const float v = s / static_cast<float>(n);     // n == 0: 0 / 0 = NaN, the mean of an empty set
    p_s[col] = v;
    if (pooled != nullptr) pooled[static_cast<int64_t>(b) * kPoolD + col] = v;
  }
  __syncthreads();
  if (logits == nullptr && probs == nullptr) return;
  // logits: warp w takes classes w, w + 8, ...; lane l sums k = 4l + 128 i (i ascending), then a fixed xor tree
  for (int c = warp; c < C; c += kHeadWarps) {
    const float4* w4 = reinterpret_cast<const float4*>(W + static_cast<int64_t>(c) * kPoolD);
    const float4* p4 = reinterpret_cast<const float4*>(p_s);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < kPoolD / 128; ++i) {
      const float4 w = __ldg(w4 + lane + 32 * i);
      const float4 p = p4[lane + 32 * i];
      acc = fmaf(w.x, p.x, acc);
      acc = fmaf(w.y, p.y, acc);
      acc = fmaf(w.z, p.z, acc);
      acc = fmaf(w.w, p.w, acc);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) l_s[c] = acc + __ldg(bias + c);
  }
  __syncthreads();
  const bool live = tid < C;
  const float v = live ? l_s[tid] : -INFINITY;
  if (live && logits != nullptr) logits[static_cast<int64_t>(b) * C + tid] = v;
  if (probs == nullptr) return;
  // softmax: block max, exp, block sum (xor tree in each warp, then the warp partials in ascending order)
  float m = v;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if (lane == 0) red_s[warp] = m;
  __syncthreads();
  m = red_s[0];
#pragma unroll
  for (int w = 1; w < kHeadWarps; ++w) m = fmaxf(m, red_s[w]);
  __syncthreads();   // red_s is reused for the sums
  float e = live ? expf(v - m) : 0.f;
  float s = e;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) red_s[warp] = s;
  __syncthreads();
  s = red_s[0];
#pragma unroll
  for (int w = 1; w < kHeadWarps; ++w) s += red_s[w];
  if (live) probs[static_cast<int64_t>(b) * C + tid] = e / s;
}

}  // namespace

void launch_pool_chunks(const float* enc, const int* enc_len, int B, int T, float* part, cudaStream_t s) {
  const int n_chunks = pool_chunk_count(T);
  pool_chunks_kernel<<<dim3(B, n_chunks), kPoolThreads, 0, s>>>(enc, enc_len, B, T, n_chunks, part);
}

void launch_pooled_head(const float* part, const int* enc_len, int B, int T, const float* W, const float* bias, int C, float* pooled,
                        float* logits, float* probs, cudaStream_t s) {
  pooled_head_kernel<<<B, kHeadThreads, 0, s>>>(part, enc_len, B, T, pool_chunk_count(T), W, bias, C, pooled, logits, probs);
}

}  // namespace gam
