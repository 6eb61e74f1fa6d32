// Tensor-core attention for the Conformer block (head_dim <= 48, any T', key-padding mask by length).
// Replaces F.scaled_dot_product_attention / flash_attn_varlen in
// gigaam/encoder.py:258-277 (RotaryPositionMultiHeadAttention) on the q/k/v produced by the fused
// LN+RoPE -> GEMM kernels.
//
//   qkv : [rows, 2304] fp16 = [q(768) | k(768) | v(768)], head h at columns h*48 .. h*48+47 of each part
//   out : [rows, 768]  fp16
//
// Rows are PACKED (the varlen contract of gigaam/utils.py:103-155, apply_masked_flash_attn): utterance b owns rows
// cu[b] .. cu[b] + klen[b]; only the query tiles and key blocks that hold one of its frames are computed, a tile that
// reaches past the utterance reads its neighbour's rows (masked as keys, never stored as queries).  With cu == null the
// layout is the padded [B, T] one (unit tests): row b*T, every query row stored.  The rows of the last key block past
// klen are zeroed in shared memory before P.V: their P is 0, but 0 x (stale inf / NaN bits) would not be.
//
// One CTA per (128-query tile, head, utterance), eight warps of 16 query rows each.  A single thread issues TMA loads of
// the Q tile and of the first min(nk, 6) K / V blocks of the utterance (32 KB each, every stage on its own mbarrier), so
// the first block's math starts while the rest are still in flight.  Up to T' = 768 that is every block and nothing is
// ever reloaded.  Longer utterances run the stages as a ring: key block kb lives in stage kb % 6, and once all eight
// warps are done with block kb (a __syncthreads after its P.V) thread 0 refills the stage with block kb + 6, which
// therefore has five blocks of math to land in.  Per key block of 128:
// S = Q K^T with mma.sync m16n8k16 (operands by ldmatrix from the SWIZZLE_128B tiles TMA wrote), an online softmax on
// the S fragment in registers, and O += P V with P re-packed from the S fragment as the A operand (no shared-memory
// round trip).  The softmax:
//   * LAZY reference point: exact block maximum on the first block; afterwards it moves only when a block maximum exceeds
//     it by more than 2^8 (P then stays <= 256, far inside fp16).  Moving it rescales O and the row sum;
//   * the denominator is the fp32 sum of exactly the fp16 P that P.V used.
#include "../../include/gigaam_b200.h"
#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace gam {
namespace {

static_assert(GAM_ROTARY_MAX_DK == 3 * 16, "launch_attention instantiates KS = 1 .. 3");

constexpr int kMaxKB = 6;             // K / V stages: 768 keys resident (30 s segments of the reference's VAD, gigaam/vad_utils.py:85)
constexpr int kTileBytes = 128 * 128;  // 128 rows x 64 fp16
constexpr int kThreads = 256;
constexpr float kLazyLog2 = 8.0f;      // the softmax reference point trails the running maximum by at most 2^8
constexpr int kBarBytes = 128;

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttnParams {
  int T, nkb;
  const int* klen;
  const int* cu;
  __half* out;
  int ld_out, dk;
  float scale_log2;
};

// KS = dk / 16
template <int KS>
__global__ void __launch_bounds__(kThreads) attention_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nst = min(p.nkb, kMaxKB);              // stages in shared memory
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTileBytes;                  // [nst]
  uint8_t* sV = sK + nst * kTileBytes;              // [nst]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + nst * kTileBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                     // [kMaxKB]

  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int klen = p.klen != nullptr ? min(max(__ldg(p.klen + b), 0), p.T) : p.T;
  const int kb_valid = (klen + 127) >> 7;
  // packed rows: a query tile past the utterance's last frame has nothing to compute or store (uniform for the CTA)
  if (p.cu != nullptr && qt >= kb_valid) return;
  const int row0 = p.cu != nullptr ? __ldg(p.cu + b) : b * p.T;
  const int qlim = p.cu != nullptr ? klen : p.T;   // query rows that are stored
  const int nk = max(1, kb_valid);                 // key blocks that are multiplied
  const int dmodel = p.ld_out;

  // key block kb -> stage kb % kMaxKB (its completion kb / kMaxKB of kv_full[stage])
  auto issue_block = [&](int kb, int st) {
    ptx::mbar_arrive_expect_tx(&kv_full[st], 2 * kTileBytes);
    ptx::tma_load_2d(sK + st * kTileBytes, &tmap_qkv, &kv_full[st], dmodel + h * p.dk, row0 + kb * 128);
    ptx::tma_load_2d(sV + st * kTileBytes, &tmap_qkv, &kv_full[st], 2 * dmodel + h * p.dk, row0 + kb * 128);
  };
  if (threadIdx.x == 0) {
    const int npre = nk < kMaxKB ? nk : kMaxKB;    // blocks issued up front, one per stage
    ptx::prefetch_tmap(&tmap_qkv);
    ptx::mbar_init(q_full, 1);
#pragma unroll
    for (int i = 0; i < kMaxKB; ++i)
      if (i < npre) ptx::mbar_init(&kv_full[i], 1);
    ptx::fence_mbar_init();
    ptx::mbar_arrive_expect_tx(q_full, kTileBytes);
    ptx::tma_load_2d(sQ, &tmap_qkv, q_full, h * p.dk, row0 + qt * 128);
#pragma unroll
    for (int kb = 0; kb < kMaxKB; ++kb)
      if (kb < npre) issue_block(kb, kb);
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  // Q fragments of this warp's 16 rows, all of dk
  uint32_t qa[KS][4];
  ptx::mbar_wait(q_full, 0);
#pragma unroll
  for (int kk = 0; kk < KS; ++kk)
    ptx::ldsm_x4(ptx::smem_u32(sQ) + ptx::sw128_off(warp * 16 + (lane & 15), kk * 16 + (lane >> 4) * 8), qa[kk][0], qa[kk][1],
                 qa[kk][2], qa[kk][3]);

  float o[2 * KS][4];
#pragma unroll
  for (int i = 0; i < 2 * KS; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float mc[2] = {0.f, 0.f};     // softmax reference point x scale (log2 domain), rows g and g + 8
  float sum[2] = {0.f, 0.f};    // this thread's share of the row sums

  for (int kb = 0; kb < nk; ++kb) {
    const int nvalid = max(min(klen - kb * 128, 128), 0);
    const int st = kb % kMaxKB;
    ptx::mbar_wait(&kv_full[st], (kb / kMaxKB) & 1);
    uint8_t* kt = sK + st * kTileBytes;
    uint8_t* vt = sV + st * kTileBytes;
    if (nvalid < 128) {   // only the last block (uniform for the CTA; its stage is never refilled): V rows past klen -> 0
      __syncthreads();
      for (int i = threadIdx.x; i < (128 - nvalid) * 8; i += kThreads)
        reinterpret_cast<uint4*>(vt + nvalid * 128)[i] = make_uint4(0u, 0u, 0u, 0u);
      __syncthreads();
    }
    const int nch = (nvalid + 15) >> 4;   // 16-key chunks that hold a valid key

    // ---- S = Q K^T for this warp's 16 rows x 128 keys
    float s[16][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[2 * j][0] = s[2 * j][1] = s[2 * j][2] = s[2 * j][3] = 0.f;
      s[2 * j + 1][0] = s[2 * j + 1][1] = s[2 * j + 1][2] = s[2 * j + 1][3] = 0.f;
      if (j < nch) {
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
          uint32_t b0, b1, b2, b3;
          ptx::ldsm_x4(ptx::smem_u32(kt) + ptx::sw128_off(16 * j + (lane & 7) + ((lane >> 4) << 3), kk * 16 + ((lane >> 3) & 1) * 8),
                       b0, b1, b2, b3);
          ptx::mma_16816(s[2 * j], qa[kk], b0, b1);
          ptx::mma_16816(s[2 * j + 1], qa[kk], b2, b3);
        }
      }
    }

    // ---- block maximum of rows g, g + 8 over the valid keys (the quad of 4 threads shares a row)
    float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (8 * i + 2 * t4 + (e & 1) < nvalid) bm[e >> 1] = fmaxf(bm[e >> 1], s[i][e]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 1));
      bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 2));
      // reference point: exact on the first block, afterwards moved only when it trails by more than 2^kLazyLog2
      const float bml = bm[r] * p.scale_log2;
      if (kb == 0) {
        mc[r] = bm[r] == -INFINITY ? 0.f : bml;
      } else if (bml > mc[r] + kLazyLog2) {
        const float corr = ex2(mc[r] - bml);
        mc[r] = bml;
        sum[r] *= corr;
#pragma unroll
        for (int i = 0; i < 2 * KS; ++i) {
          o[i][2 * r] *= corr;
          o[i][2 * r + 1] *= corr;
        }
      }
    }

    // ---- p = exp2(s * scale - reference) -> fp16, and O += P V per 16-key chunk
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < nch) {
        uint32_t pa[4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int key = 16 * j + 8 * u + 2 * t4;
            const float p0 = key < nvalid ? ex2(fmaf(s[2 * j + u][2 * r], p.scale_log2, -mc[r])) : 0.f;
            const float p1 = key + 1 < nvalid ? ex2(fmaf(s[2 * j + u][2 * r + 1], p.scale_log2, -mc[r])) : 0.f;
            const __half2 hh = __floats2half2_rn(p0, p1);
            const float2 pr = __half22float2(hh);
            sum[r] += pr.x + pr.y;
            pa[2 * u + r] = *reinterpret_cast<const uint32_t*>(&hh);
          }
        }
#pragma unroll
        for (int dd = 0; dd < KS; ++dd) {
          uint32_t b0, b1, b2, b3;
          ptx::ldsm_x4_t(ptx::smem_u32(vt) + ptx::sw128_off(16 * j + (lane & 7) + (((lane >> 3) & 1) << 3), dd * 16 + ((lane >> 4) << 3)),
                         b0, b1, b2, b3);
          ptx::mma_16816(o[2 * dd], pa, b0, b1);
          ptx::mma_16816(o[2 * dd + 1], pa, b2, b3);
        }
      }
    }
    // every warp is done with this stage (K in S = QK^T, V in P.V): refill it with block kb + kMaxKB
    if (kb + kMaxKB < nk) {
      __syncthreads();
      if (threadIdx.x == 0) issue_block(kb + kMaxKB, st);
    }
  }

  // ---- O / row sum -> fp16 (a row without a valid key: sum 0 -> zeros)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
    const float inv = sum[r] > 0.f ? 1.0f / sum[r] : 0.f;
    const int q = qt * 128 + warp * 16 + g + 8 * r;
    if (q < qlim) {
      __half* dst = p.out + (static_cast<size_t>(row0) + q) * p.ld_out + h * p.dk + 2 * t4;
#pragma unroll
      for (int i = 0; i < 2 * KS; ++i) {
        const __half2 hh = __floats2half2_rn(o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
        *reinterpret_cast<__half2*>(dst + 8 * i) = hh;
      }
    }
  }
}

template <int KS>
int launch_ks(const CUtensorMap* tmap_qkv, const AttnParams& p, int B, int H, cudaStream_t s) {
  const int smem = (1 + 2 * (p.nkb < kMaxKB ? p.nkb : kMaxKB)) * kTileBytes + kBarBytes + 1024;
  static PerDeviceOnce attr_once;
  if (attr_once.first() &&
      cudaFuncSetAttribute(attention_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (1 + 2 * kMaxKB) * kTileBytes + kBarBytes + 1024) !=
          cudaSuccess)
    return -2;
  return launch_k(attention_kernel<KS>, dim3(p.nkb, H, B), dim3(kThreads), smem, s, *tmap_qkv, p) == cudaSuccess ? 0 : -2;
}

}  // namespace

int launch_attention(const CUtensorMap* tmap_qkv, const int* klen, const int* cu, __half* out, int B, int T, int H, int dk,
                     int d_model, cudaStream_t s) {
  const int nkb = (T + 127) / 128;
  if (nkb <= 0 || dk % 16 != 0 || dk > GAM_ROTARY_MAX_DK || (cu != nullptr && klen == nullptr)) return -1;
  AttnParams p;
  p.T = T;
  p.nkb = nkb;
  p.klen = klen;
  p.cu = cu;
  p.out = out;
  p.ld_out = d_model;
  p.dk = dk;
  p.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(dk));
  switch (dk / 16) {
    case 1: return launch_ks<1>(tmap_qkv, p, B, H, s);
    case 2: return launch_ks<2>(tmap_qkv, p, B, H, s);
    default: return launch_ks<3>(tmap_qkv, p, B, H, s);
  }
}

}  // namespace gam
