// fp32 encoder projection of the RNN-T joint (gigaam/decoder.py:41-47: joint.enc), hoisted out of the greedy loop as one
// GEMM over all frames; the loop itself lives in rnnt_cluster.cu.  The joint lattice (heads.cu) uses the same GEMM for
// both of its projections.  All head arithmetic stays fp32 (the reference never casts the head to fp16,
// gigaam/__init__.py:188-189).
#include "kernels.h"

namespace gam {
namespace {

// ------------------------------------------------------------------ fp32 GEMM  C[M,N] = A[M,K] W[N,K]^T + bias
// W_KN: W is given transposed, as Wt[K,N] row-major (N % 4 == 0), e.g. rnnt_wp_t.  Either way every C element sums over k
// in ascending order.
constexpr int kSgBM = 64, kSgBN = 64, kSgBK = 16;
template <bool W_KN>
__global__ void __launch_bounds__(256) sgemm_bias_kernel(const float* __restrict__ A, const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ C, int M,
                                                            int N, int K) {
  __shared__ float As[kSgBK][kSgBM + 4];
  __shared__ float Ws[kSgBK][kSgBN + 4];
  const int m0 = blockIdx.y * kSgBM, n0 = blockIdx.x * kSgBN;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += kSgBK) {
    {
      const int r = threadIdx.x / 4, k4 = (threadIdx.x % 4) * 4;
      float4 a = make_float4(0, 0, 0, 0), w = make_float4(0, 0, 0, 0);
      if (m0 + r < M) a = *reinterpret_cast<const float4*>(A + static_cast<size_t>(m0 + r) * K + k0 + k4);
      As[k4 + 0][r] = a.x; As[k4 + 1][r] = a.y; As[k4 + 2][r] = a.z; As[k4 + 3][r] = a.w;
      if constexpr (W_KN) {
        const int k = threadIdx.x / 16, n4 = (threadIdx.x % 16) * 4;
        if (n0 + n4 < N) w = *reinterpret_cast<const float4*>(W + static_cast<size_t>(k0 + k) * N + n0 + n4);
        Ws[k][n4 + 0] = w.x; Ws[k][n4 + 1] = w.y; Ws[k][n4 + 2] = w.z; Ws[k][n4 + 3] = w.w;
      } else {
        if (n0 + r < N) w = *reinterpret_cast<const float4*>(W + static_cast<size_t>(n0 + r) * K + k0 + k4);
        Ws[k4 + 0][r] = w.x; Ws[k4 + 1][r] = w.y; Ws[k4 + 2][r] = w.z; Ws[k4 + 3][r] = w.w;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSgBK; ++k) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; w[i] = Ws[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < N) C[static_cast<size_t>(m) * N + n] = acc[i][j] + (bias ? bias[n] : 0.f);
    }
  }
}

}  // namespace

void launch_sgemm_tn_bias(const float* A, const float* W, const float* bias, float* C, int M, int N, int K, cudaStream_t s) {
  dim3 grid((N + kSgBN - 1) / kSgBN, (M + kSgBM - 1) / kSgBM);
  sgemm_bias_kernel<false><<<grid, 256, 0, s>>>(A, W, bias, C, M, N, K);
}
void launch_sgemm_nn_bias(const float* A, const float* Wt, const float* bias, float* C, int M, int N, int K, cudaStream_t s) {
  dim3 grid((N + kSgBN - 1) / kSgBN, (M + kSgBM - 1) / kSgBM);
  sgemm_bias_kernel<true><<<grid, 256, 0, s>>>(A, Wt, bias, C, M, N, K);
}

}  // namespace gam
