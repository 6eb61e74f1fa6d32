// Instantiations and host launchers of the wgmma GEMM (gemm_sm90.cuh: 128 x 256 tiles, persistent clusters of two CTAs).
#include <climits>
#include <cstdlib>

#include "gemm_sm90.cuh"
#include "kernels.h"
#include "launch.cuh"

namespace gam {
namespace {

constexpr int kBN = kG2BN;

// p.num_m_tiles counts 128-row blocks; the grid is one cluster of kG2Cluster CTAs per co-resident pair of m-blocks
// (max_clusters: gemm_init's count), each walking the list of tile pairs
// to: output map of the shared-memory store path (gemm_sm90.cuh); without it (null) every tile stores straight from the
// fragment
template <int EPI, int AMODE>
int launch_v2(const CUtensorMap* ta, const CUtensorMap* tw, GemmParams p, int max_clusters, cudaStream_t s,
              const CUtensorMap* ta2 = nullptr, const CUtensorMap* to = nullptr) {
  auto kern = gemm_f16_tn_kernel<EPI, AMODE>;
  const int pairs = (p.num_m_tiles + kG2Cluster - 1) / kG2Cluster * p.num_n_tiles;
  const int nclusters = pairs < max_clusters ? pairs : max_clusters;
  if (nclusters <= 0) return 0;
  p.tma_out = gemm_tma_store<EPI, AMODE>() && to != nullptr;
  return launch_k(kern, dim3(nclusters * kG2Cluster), dim3(kG2Threads), gemm_smem_bytes<EPI, AMODE>(), s, *ta, ta2 ? *ta2 : *ta, *tw, to ? *to : *ta,
                  p) == cudaSuccess
             ? 0
             : -2;
}

// opt in to the dynamic shared memory and lower *clusters to the number of this instantiation's clusters that fit
// on the current device at once
template <int EPI, int AMODE>
int init_one(int* clusters) {
  auto kern = gemm_f16_tn_kernel<EPI, AMODE>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, gemm_smem_bytes<EPI, AMODE>()) != cudaSuccess)
    return -1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(kG2Cluster);
  cfg.blockDim = dim3(kG2Threads);
  cfg.dynamicSmemBytes = gemm_smem_bytes<EPI, AMODE>();
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) return -1;
  if (n < *clusters) *clusters = n;
  return 0;
}

}  // namespace

int gemm_init(int* max_clusters) {
  int n = INT_MAX, rc = 0;
  rc |= init_one<EPI_BIAS_F16, A_2D>(&n);
  rc |= init_one<EPI_BIAS_SILU_F16, A_2D>(&n);
  rc |= init_one<EPI_BIAS_GLU_F16, A_2D>(&n);
  rc |= init_one<EPI_BIAS_RES_F32, A_2D>(&n);
  rc |= init_one<EPI_BIAS_F32, A_2D>(&n);
  rc |= init_one<EPI_CONV_RELU_MASK_F16, A_CONV>(&n);
  rc |= init_one<EPI_POWER_F32, A_2D>(&n);
  rc |= init_one<EPI_CONV_RELU_MASK_F16, A_CONV1D>(&n);
  rc |= init_one<EPI_CONV_RELU_MASK_F32, A_CONV1D>(&n);
  *max_clusters = n;
  return rc;
}

int launch_gemm(int kind, const CUtensorMap* ta, const CUtensorMap* tw, int M, int N, int K, const float* bias,
                const float* res, void* out, int ldo, float scale, int max_clusters, cudaStream_t s, int reverse, const int* m_dev,
                const CUtensorMap* to) {
  if (N % kBN != 0 || K % kGemmBK != 0 || M <= 0) return -1;
  GemmParams p{};
  p.M = M;
  p.m_dev = m_dev;
  p.N = N;
  p.num_m_tiles = (M + kGemmBM - 1) / kGemmBM;
  p.num_n_tiles = N / kBN;
  p.num_k_blocks = K / kGemmBK;
  p.bias = bias;
  p.res = res;
  p.out = out;
  p.ldo = ldo;
  p.scale = scale;
  p.reverse = reverse;
  switch (kind) {
    case GEMM_BIAS_F16: return launch_v2<EPI_BIAS_F16, A_2D>(ta, tw, p, max_clusters, s, nullptr, to);
    case GEMM_BIAS_SILU_F16: return launch_v2<EPI_BIAS_SILU_F16, A_2D>(ta, tw, p, max_clusters, s, nullptr, to);
    case GEMM_BIAS_GLU_F16: return launch_v2<EPI_BIAS_GLU_F16, A_2D>(ta, tw, p, max_clusters, s, nullptr, to);
    case GEMM_BIAS_RES_F32: return launch_v2<EPI_BIAS_RES_F32, A_2D>(ta, tw, p, max_clusters, s);
    case GEMM_BIAS_F32: return launch_v2<EPI_BIAS_F32, A_2D>(ta, tw, p, max_clusters, s, nullptr, to);
    default: return -1;
  }
}

// D[:, :n1] = A1 W[:n1]^T + b, D[:, n1:] = A2 W[n1:]^T + b  (fp16 out) in ONE launch of the persistent kernel: more tiles
// per launch = less wave quantisation and one launch less.
int launch_gemm_dual_a(const CUtensorMap* ta1, const CUtensorMap* ta2, int n1, const CUtensorMap* tw, int M, int N, int K,
                       const float* bias, void* out, int ldo, int max_clusters, cudaStream_t s, int reverse, const int* m_dev,
                       const CUtensorMap* to) {
  if (N % kBN != 0 || n1 % kBN != 0 || n1 <= 0 || n1 >= N || K % kGemmBK != 0 || M <= 0) return -1;
  GemmParams p{};
  p.M = M;
  p.m_dev = m_dev;
  p.N = N;
  p.num_m_tiles = (M + kGemmBM - 1) / kGemmBM;
  p.num_n_tiles = N / kBN;
  p.num_k_blocks = K / kGemmBK;
  p.bias = bias;
  p.out = out;
  p.ldo = ldo;
  p.scale = 1.f;
  p.a1_nblks = n1 / kBN;
  p.reverse = reverse;
  return launch_v2<EPI_BIAS_F16, A_2D>(ta1, tw, p, max_clusters, s, ta2, to);
}

int launch_gemm_conv(const CUtensorMap* ta4, const CUtensorMap* tw, int B, int T2, int C, int N, const float* bias,
                     const int* len2, const int* cu, const int* plen, void* out, int ldo, int max_clusters, cudaStream_t s) {
  if (N % kBN != 0 || C % kGemmBK != 0 || (cu != nullptr) != (plen != nullptr)) return -1;
  GemmParams p{};
  p.M = 0;
  p.conv_cu = cu;
  p.conv_plen = plen;
  p.N = N;
  p.conv_T2 = T2;
  p.conv_tiles_per_utt = (T2 + 7) / 8;
  p.conv_kchunks = C / kGemmBK;
  p.conv_len2 = len2;
  p.conv_num_blocks = B * p.conv_tiles_per_utt;
  p.num_m_tiles = p.conv_num_blocks;
  p.num_n_tiles = N / kBN;
  p.num_k_blocks = 9 * p.conv_kchunks;
  p.bias = bias;
  p.res = nullptr;
  p.out = out;
  p.ldo = ldo;
  p.scale = 1.f;
  return launch_v2<EPI_CONV_RELU_MASK_F16, A_CONV>(ta4, tw, p, max_clusters, s);
}

// power spectrum of a split-precision DFT: D = A W^T with W tiles [128 cos | 128 sin]; out[:, N/2] = re^2 + im^2
int launch_gemm_power(const CUtensorMap* ta, const CUtensorMap* tw, int M, int N, int K, float* out, int ldo, int max_clusters,
                      cudaStream_t s) {
  if (N % kBN != 0 || K % kGemmBK != 0 || M <= 0) return -1;
  GemmParams p{};
  p.M = M;
  p.N = N;
  p.num_m_tiles = (M + kGemmBM - 1) / kGemmBM;
  p.num_n_tiles = N / kBN;
  p.num_k_blocks = K / kGemmBK;
  p.out = out;
  p.ldo = ldo;
  p.scale = 1.0f / (2048.0f * 2048.0f * 8.0f * 8.0f);   // frames x 2^11, basis x 2^3 (engine.py DFT_*_SCALE), squared
  return launch_v2<EPI_POWER_F32, A_2D>(ta, tw, p, max_clusters, s);
}

// k-tap / stride-2 conv1d over time-major [B, T_in, C_in] as an implicit GEMM (3-D strided TMA), K order (tap, c).
// out rows = (b, t_out); fp16 (intermediate stage) or fp32 (last stage = encoder input) with ReLU + time mask.
int launch_gemm_conv1d(const CUtensorMap* ta3, const CUtensorMap* tw, int B, int T_out, int C_in, int taps, int N,
                       const float* bias, const int* len_out, const int* cu, const int* plen, void* out, int ldo, int f32_out,
                       int max_clusters, cudaStream_t s) {
  if (N % kBN != 0 || C_in % kGemmBK != 0 || taps < 1 || (cu != nullptr) != (plen != nullptr)) return -1;
  GemmParams p{};
  p.conv_cu = cu;
  p.conv_plen = plen;
  p.N = N;
  p.conv_T2 = T_out;
  p.conv_tiles_per_utt = (T_out + 127) / 128;
  p.conv_kchunks = C_in / kGemmBK;
  p.conv_len2 = len_out;
  p.conv_num_blocks = B * p.conv_tiles_per_utt;
  p.conv_pad = (taps - 1) / 2;
  p.num_m_tiles = p.conv_num_blocks;
  p.num_n_tiles = N / kBN;
  p.num_k_blocks = taps * p.conv_kchunks;
  p.bias = bias;
  p.out = out;
  p.ldo = ldo;
  p.scale = 1.f;
  return f32_out ? launch_v2<EPI_CONV_RELU_MASK_F32, A_CONV1D>(ta3, tw, p, max_clusters, s)
                 : launch_v2<EPI_CONV_RELU_MASK_F16, A_CONV1D>(ta3, tw, p, max_clusters, s);
}

}  // namespace gam
