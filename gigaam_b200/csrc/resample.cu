// Polyphase resampling to 16 kHz (include/gigaam_b200.h, gam_resample): torchaudio's default sinc_interp_hann resampler,
//   y[j n + p] = sum_k h[p, k] x[j o + k - w],  k = 0 .. K-1,  K = 2 w + o,
// with o / n the reduced rate ratio and samples outside a row's input span read as zero.
//
// One thread per output, consecutive outputs across a warp.  The table is stored k-major ([K, n]), so at a given tap the
// lanes of a warp, which hold consecutive phases p, read consecutive words; their input samples are the same word (n > 1)
// or o words apart (n = 1).  Both go through the read-only path; the table (at most 4 MiB) and an output tile's input span
// stay in L1 / L2.
//
// Summation order: every output is one chain of fp32 FMAs over k in increasing order, started from +0.  Taps whose sample
// lies outside the span are zero, and the loop skips them: an FMA with a zero product leaves a chain that started at +0
// unchanged (the chain can never hold -0, since x + y rounds to -0 only when both are -0), so skipping them gives the same
// bits as adding them.  An output therefore depends on its own span of inputs only, whatever batch, chunk or launch it is
// computed in.
#include "kernels.h"

namespace gam {
namespace {

constexpr int kResampleThreads = 256;

__global__ void __launch_bounds__(kResampleThreads)
    resample_kernel(const float* __restrict__ x, int64_t x_pitch, const float* __restrict__ table, int n, int o, int w, int K,
                    const int64_t* __restrict__ spans, int B, float* __restrict__ y, int64_t y_pitch) {
  const int b = blockIdx.y;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kResampleThreads + threadIdx.x;
  const int64_t in_lo = spans[b], out_lo = spans[2 * B + b], out_hi = spans[3 * B + b];
  const int64_t in_hi = min(spans[B + b], in_lo + x_pitch);   // a row holds at most x_pitch samples
  const int64_t m = out_lo + i;
  if (i >= y_pitch || m >= out_hi || m < 0) return;
  const int64_t j = m / n;
  const int p = static_cast<int>(m - j * n);
  const int64_t first = j * o - w;   // input sample of tap 0
  const int k0 = static_cast<int>(min(max(in_lo - first, int64_t(0)), int64_t(K)));
  const int k1 = static_cast<int>(min(max(in_hi - first, int64_t(0)), int64_t(K)));
  const float* xr = x + b * x_pitch + (first - in_lo);
  const float* hp = table + p;
  float acc = 0.0f;
  for (int k = k0; k < k1; ++k) acc = fmaf(__ldg(hp + static_cast<int64_t>(k) * n), __ldg(xr + k), acc);
  y[b * y_pitch + i] = acc;
}

}  // namespace

void launch_resample(const float* x, int64_t x_pitch, const float* table, int n, int o, int w, int K, const int64_t* spans, int B,
                     float* y, int64_t y_pitch, cudaStream_t s) {
  const dim3 grid(static_cast<unsigned>((y_pitch + kResampleThreads - 1) / kResampleThreads), static_cast<unsigned>(B));
  resample_kernel<<<grid, kResampleThreads, 0, s>>>(x, x_pitch, table, n, o, w, K, spans, B, y, y_pitch);
}

}  // namespace gam
