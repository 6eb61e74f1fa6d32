// Shared definitions of the wgmma GEMM (gemm_sm90.cuh): epilogue / A-operand modes, the parameter block, and the
// small math helpers of the fused epilogues.
//
//   * A and W are fp16, K-contiguous ("TN"): exactly the layout of an activation matrix [rows, feat]
//     and of an nn.Linear / Conv1d(k=1) weight [out, in] (reference: gigaam/encoder.py:145-148,
//     378,393,418-420), so no operand is ever transposed in memory.
//   * A_CONV mode: the A operand is the implicit im2col of a channels-last activation
//     [B, T1, F1, C] for a 3x3 / stride-2 / pad-1 convolution (reference: gigaam/encoder.py:59-70),
//     fetched tap by tap with a 4-D strided TMA box (elementStrides = 2 on T and F, OOB = zero fill
//     = the conv's zero padding).  Nothing is ever materialised as an im2col matrix.
#pragma once
#include "ptx.cuh"

namespace gam {

enum GemmEpilogue : int {
  EPI_BIAS_F16 = 0,        // out16 = acc + bias
  EPI_BIAS_SILU_F16 = 1,   // out16 = silu(acc + bias)
  EPI_BIAS_GLU_F16 = 2,    // out16[:, n] = (acc_a + bias_a) * sigmoid(acc_b + bias_b), tile = [a|b]
  EPI_BIAS_RES_F32 = 3,    // out32 = res + scale * (acc + bias)
  EPI_BIAS_F32 = 4,        // out32 = acc + bias
  EPI_CONV_RELU_MASK_F16 = 5,  // out16 = t2 < len2[b] ? relu(acc + bias) : 0   (A_CONV / A_CONV1D row mapping)
  EPI_CONV_RELU_MASK_F32 = 6,  // out32 = t < len[b] ? relu(acc + bias) : 0      (A_CONV1D, last subsampling stage)
  EPI_POWER_F32 = 7,           // out32[:, n] = re^2 + im^2, tile = [128 re | 128 im]  (DFT power spectrum, no bias)
};

// A_CONV  : implicit im2col of a 3x3 / stride-2 conv2d over channels-last [B, T1, F1, C]  (4-D strided TMA)
// A_CONV1D: implicit im2col of a k-tap / stride-2 conv1d over time-major [B, T_in, C]      (3-D strided TMA);
//           a 128-row block = 128 consecutive output frames of one utterance
enum GemmAMode : int { A_2D = 0, A_CONV = 1, A_CONV1D = 2 };

struct GemmParams {
  int M;             // valid rows of D (A_2D) ; unused for A_CONV
  int N;             // columns of the accumulator matrix (= rows of W)
  int num_m_tiles;
  int num_n_tiles;
  int num_k_blocks;  // K / 64   (A_CONV: 9 taps * C/64)
  const float* bias;  // [N] in accumulator column order
  const float* res;   // fp32 residual, row pitch ldo (EPI_BIAS_RES_F32)
  void* out;
  int ldo;            // output row pitch in elements
  float scale;
  // A_CONV only
  int conv_T2;            // output time steps per utterance
  int conv_tiles_per_utt; // ceil(T2 / 8)
  int conv_kchunks;       // C / 64
  int conv_num_blocks;    // B * conv_tiles_per_utt  (128-row blocks that exist)
  int conv_pad;           // A_CONV1D: (taps - 1) / 2
  const int* conv_len2;   // [B] valid output time steps
  // A_2D only: n-tiles [0, a1_nblks) read A through tmap_a, the rest through tmap_a2 (0 = tmap_a for all).
  // Lets two GEMMs that share M, K and the output buffer but not the A operand (W_qk on rope(u), W_v on u) run as one launch.
  int a1_nblks;
  // Packed (varlen) rows.  After the subsampling the encoder keeps only the frames that exist: utterance b owns rows
  // cu[b] .. cu[b] + plen[b] of every activation matrix and the row count is known on the device only (lengths arrive as a
  // device tensor and the step may be a replayed CUDA graph) -- flash_attn_varlen's cu_seqlens contract
  // (gigaam/utils.py:103-155) applied to the whole block instead of the attention alone.
  const int* m_dev;       // A_2D: valid rows of D read on the device (null: M); the grid is sized for M = the padded maximum
  const int* conv_cu;     // conv modes: output row of frame (b, t) = conv_cu[b] + t (null: b * conv_T2 + t, all conv_T2 frames)
  const int* conv_plen;   // conv modes with conv_cu: frames t < conv_plen[b] exist; row blocks past it are skipped entirely
  // A_2D only: walk the tiles from the last row block to the first.  Consecutive kernels of a layer alternate direction
  // (gam_api.cu): a consumer then starts on the rows its producer wrote LAST, which are the ones still in the 50 MB L2 --
  // read in the producer's own order, a buffer that does not fit is evicted just ahead of the reader (LRU) and every
  // byte comes from DRAM.
  int reverse;
  // A_2D epilogues but EPI_BIAS_RES_F32 and EPI_POWER_F32: tiles whose 128 rows all lie below the live row count leave
  // through shared memory and TMA bulk stores (tmap_out); 0 = every tile stores directly from the fragment (the output
  // could not be described by a tensor map)
  int tma_out;
};

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;
__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// silu(x) = x * sigmoid(x) = 0.5x * (1 + tanh(0.5x))
__device__ __forceinline__ float silu_f(float x) {
  float h = 0.5f * x;
  return fmaf(h, fast_tanh(h), h);
}
__device__ __forceinline__ float sigmoid_f(float x) { return fmaf(0.5f, fast_tanh(0.5f * x), 0.5f); }

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}


}  // namespace gam
