// Tensor-core attention with Transformer-XL relative positions (v1_* checkpoints, self_attention_model == "rel_pos").
// Replaces RelPositionMultiHeadAttention.forward (gigaam/encoder.py:208-228) + forward_attention (:173-188) on
// the output of ONE projection GEMM whose weight is [W_q ; W_q ; W_k ; W_v] and whose bias carries pos_bias_u / _v:
//
//   qkv : [rows, 4*768] fp16 = [q+u | q+v | k | v], head h at columns h*48 .. h*48+47 of each part; rows are packed
//         (utterance b = rows cu[b] .. cu[b] + klen[b]; cu == null: the padded [B, T] layout of the unit tests)
//   pos : [2*max_t-1, 768] fp16 = W_pos pe(r) for r = max_t-1 ... -(max_t-1)   (row = max_t-1-r); max_t >= T is the
//         handle's max_encoded_frames (GAM_REL_POS_MAX_T = 768 unless the model asked for more)
//   out : [rows, 768] fp16
//
//   s[i, j] = ((q_i+u) . k_j + (q_i+v) . p_{i-j}) / sqrt(d_k)          p_r = pos row for relative position r
//
// The reference materialises (q+v) P^T for all 2T-1 positions and re-indexes it with the pad/view "rel_shift"
// (:202-206).  Here, for a tile of 128 queries x 128 keys, the positions that can occur are the 255 consecutive
// table rows i0-j0-127 .. i0-j0+127 (a 256-row window loaded with the key block), and score (r, c) reads window row
// c - r + 127.  A warp owns 16 query rows; for a chunk of 16 keys its rows need only 31 consecutive window rows, so it
// multiplies (q+v) by those 32 rows (mma.sync), bounces the 16 x 32 result through a private shared-memory tile and reads
// each score's own diagonal back.
//
// One CTA per (128-query tile, head, utterance), eight warps; single sweep with a running maximum (O rescaled in
// registers).  One thread issues TMA loads of Q(u), Q(v) and a 2-stage ring of {K, V, 256 window rows} per key block;
// a stage is refilled once every warp is done with it.
//
// Window rows outside the table are zero-filled by TMA.  Past its end (row > 2*max_t-2: r < -(max_t-1)) they only meet
// keys j > i + max_t - 1 >= T, which are masked.  Before its start (row < 0: r > max_t-1, which happens in the last query
// tile when max_t is not a multiple of 128, e.g. 5000 = 39*128 + 8) they only meet queries i > j + max_t - 1 >= T, whose
// rows are never stored.
#include "../../include/gigaam_b200.h"
#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace gam {
namespace {

static_assert(GAM_REL_POS_MAX_DK == 4 * 16, "launch_attention_relpos instantiates KS = 1 .. 4");

constexpr int kThreads = 256;
constexpr int kTile = 128 * 128;         // bytes of a 128-row x 64-column fp16 tile
constexpr int kStageBytes = 4 * kTile;   // K, V, 2 position tiles
constexpr int kBdPitch = 33;             // floats per row of a warp's 16 x 32 bounce tile
constexpr int kBdBytes = 8 * 16 * kBdPitch * 4;
constexpr int kSmemBytes = 2 * kTile + 2 * kStageBytes + kBdBytes + 64 + 1024;

struct RelParams {
  int T;
  const int* klen;   // may be null
  const int* cu;     // may be null (padded rows)
  __half* out;
  int ld_out;        // d_model
  int dk;
  int pos_center;    // table row of relative position 0 (= max_t - 1)
  float scale_log2;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// KS = dk / 16
template <int KS>
__global__ void __launch_bounds__(kThreads, 1) attention_relpos_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                                                                      const __grid_constant__ CUtensorMap tmap_pos,
                                                                      const RelParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQu = smem;
  uint8_t* sQv = smem + kTile;
  uint8_t* sStage = smem + 2 * kTile;             // 2 x {K, V, Pw0, Pw1}
  float* sBd = reinterpret_cast<float*>(sStage + 2 * kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sBd) + kBdBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;    // [2]

  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  int klen = p.T;
  if (p.klen != nullptr) klen = min(max(__ldg(p.klen + b), 0), p.T);
  // packed rows: a query tile past the utterance's last frame has nothing to compute or store (uniform for the CTA)
  if (p.cu != nullptr && q0 >= klen) return;
  const int row0 = p.cu != nullptr ? __ldg(p.cu + b) : b * p.T;
  const int qlim = p.cu != nullptr ? klen : p.T;   // query rows that are stored
  const int dmodel = p.ld_out;
  const int nkb = (klen + 127) >> 7;   // key blocks that hold at least one valid key

  // block kb -> stage kb & 1: K, V and the 256 window rows; window row w holds relative position (q0 + 127 - kb*128) - w
  auto issue_block = [&](int kb) {
    const int st = kb & 1;
    uint8_t* base = sStage + st * kStageBytes;
    ptx::mbar_arrive_expect_tx(&kv_full[st], kStageBytes);
    ptx::tma_load_2d(base, &tmap_qkv, &kv_full[st], 2 * dmodel + h * p.dk, row0 + kb * 128);
    ptx::tma_load_2d(base + kTile, &tmap_qkv, &kv_full[st], 3 * dmodel + h * p.dk, row0 + kb * 128);
    const int prow = p.pos_center - (q0 + 127) + kb * 128;
    ptx::tma_load_2d(base + 2 * kTile, &tmap_pos, &kv_full[st], h * p.dk, prow);
    ptx::tma_load_2d(base + 3 * kTile, &tmap_pos, &kv_full[st], h * p.dk, prow + 128);
  };
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_qkv);
    ptx::prefetch_tmap(&tmap_pos);
    ptx::mbar_init(q_full, 1);
    ptx::mbar_init(&kv_full[0], 1);
    ptx::mbar_init(&kv_full[1], 1);
    ptx::fence_mbar_init();
    if (nkb > 0) {
      ptx::mbar_arrive_expect_tx(q_full, 2 * kTile);
      ptx::tma_load_2d(sQu, &tmap_qkv, q_full, h * p.dk, row0 + q0);
      ptx::tma_load_2d(sQv, &tmap_qkv, q_full, dmodel + h * p.dk, row0 + q0);
      for (int kb = 0; kb < nkb && kb < 2; ++kb) issue_block(kb);
    }
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  float* bd_tile = sBd + warp * 16 * kBdPitch;
  uint32_t qu[KS][4], qv[KS][4];
  float o[2 * KS][4];
#pragma unroll
  for (int i = 0; i < 2 * KS; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};

  if (nkb > 0) {
    ptx::mbar_wait(q_full, 0);
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      const uint32_t off = ptx::sw128_off(warp * 16 + (lane & 15), kk * 16 + (lane >> 4) * 8);
      ptx::ldsm_x4(ptx::smem_u32(sQu) + off, qu[kk][0], qu[kk][1], qu[kk][2], qu[kk][3]);
      ptx::ldsm_x4(ptx::smem_u32(sQv) + off, qv[kk][0], qv[kk][1], qv[kk][2], qv[kk][3]);
    }
  }

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb & 1;
    uint8_t* kt = sStage + st * kStageBytes;
    uint8_t* vt = kt + kTile;
    uint8_t* pw = kt + 2 * kTile;
    ptx::mbar_wait(&kv_full[st], (kb >> 1) & 1);
    const int nvalid = min(klen - kb * 128, 128);
    if (nvalid < 128) {   // only the last block (uniform for the CTA): V rows past klen -> 0
      __syncthreads();
      for (int i = threadIdx.x; i < (128 - nvalid) * 8; i += kThreads)
        reinterpret_cast<uint4*>(vt + nvalid * 128)[i] = make_uint4(0u, 0u, 0u, 0u);
      __syncthreads();
    }
    const int nch = (nvalid + 15) >> 4;

    // ---- s = (q+u) k + shifted (q+v) p, per 16-key chunk
    float s[16][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int u = 0; u < 2; ++u) s[2 * j + u][0] = s[2 * j + u][1] = s[2 * j + u][2] = s[2 * j + u][3] = 0.f;
      if (j < nch) {
        float bd[4][4];
#pragma unroll
        for (int n = 0; n < 4; ++n) bd[n][0] = bd[n][1] = bd[n][2] = bd[n][3] = 0.f;
        const int wb = 16 * j - 16 * warp + 112;   // first window row the chunk needs for this warp's rows
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
          uint32_t b0, b1, b2, b3;
          const int kc = kk * 16 + ((lane >> 3) & 1) * 8;
          ptx::ldsm_x4(ptx::smem_u32(kt) + ptx::sw128_off(16 * j + (lane & 7) + ((lane >> 4) << 3), kc), b0, b1, b2, b3);
          ptx::mma_16816(s[2 * j], qu[kk], b0, b1);
          ptx::mma_16816(s[2 * j + 1], qu[kk], b2, b3);
#pragma unroll
          for (int hw = 0; hw < 2; ++hw) {
            ptx::ldsm_x4(ptx::smem_u32(pw) + ptx::sw128_off(wb + 16 * hw + (lane & 7) + ((lane >> 4) << 3), kc), b0, b1, b2, b3);
            ptx::mma_16816(bd[2 * hw], qv[kk], b0, b1);
            ptx::mma_16816(bd[2 * hw + 1], qv[kk], b2, b3);
          }
        }
        // bd[row lr][x] = window row wb + x; score (lr, lc) of the chunk reads x = lc - lr + 15
#pragma unroll
        for (int n = 0; n < 4; ++n) {
#pragma unroll
          for (int e = 0; e < 4; ++e) bd_tile[(g + 8 * (e >> 1)) * kBdPitch + 8 * n + 2 * t4 + (e & 1)] = bd[n][e];
        }
        __syncwarp();
#pragma unroll
        for (int u = 0; u < 2; ++u) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int lr = g + 8 * (e >> 1), lc = 8 * u + 2 * t4 + (e & 1);
            s[2 * j + u][e] += bd_tile[lr * kBdPitch + lc - lr + 15];
          }
        }
        __syncwarp();
      }
    }

    // ---- running maximum, p = exp2((s - m) * scale) -> fp16, O += P V
    float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (8 * i + 2 * t4 + (e & 1) < nvalid) bm[e >> 1] = fmaxf(bm[e >> 1], s[i][e]);
    }
    float mc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 1));
      bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 2));
      const float m_new = fmaxf(m[r], bm[r]);
      mc[r] = m_new * p.scale_log2;
      const float corr = ex2(fmaf(m[r], p.scale_log2, -mc[r]));   // m == -inf on the first block -> 0
      sum[r] *= corr;
#pragma unroll
      for (int i = 0; i < 2 * KS; ++i) {
        o[i][2 * r] *= corr;
        o[i][2 * r + 1] *= corr;
      }
      m[r] = m_new;
    }
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
            const float2 pr = __half22float2(hh);   // the denominator sums exactly the fp16 P that P.V uses
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
    // every warp is done with this stage: refill it with block kb + 2
    if (kb + 2 < nkb) {
      __syncthreads();
      if (threadIdx.x == 0) issue_block(kb + 2);
    }
  }

  // ---- O / sum -> fp16 (an utterance without a single valid key gets zeros)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
    const float inv = sum[r] > 0.f ? 1.0f / sum[r] : 0.f;
    const int q = q0 + warp * 16 + g + 8 * r;
    if (q < qlim) {
      __half* dst = p.out + (static_cast<size_t>(row0) + q) * p.ld_out + h * p.dk + 2 * t4;
#pragma unroll
      for (int i = 0; i < 2 * KS; ++i)
        *reinterpret_cast<__half2*>(dst + 8 * i) = __floats2half2_rn(o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
    }
  }
}

template <int KS>
int launch_ks(const CUtensorMap* tmap_qkv, const CUtensorMap* tmap_pos, const RelParams& p, int nkb, int B, int H, cudaStream_t s) {
  static PerDeviceOnce attr_once;
  if (attr_once.first() &&
      cudaFuncSetAttribute(attention_relpos_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
    return -2;
  return launch_k(attention_relpos_kernel<KS>, dim3(nkb, H, B), dim3(kThreads), kSmemBytes, s, *tmap_qkv, *tmap_pos, p) ==
                 cudaSuccess
             ? 0
             : -2;
}

}  // namespace

int launch_attention_relpos(const CUtensorMap* tmap_qkv, const CUtensorMap* tmap_pos, int max_t, const int* klen, const int* cu,
                            __half* out, int B, int T, int H, int dk, int d_model, cudaStream_t s) {
  const int nkb = (T + 127) / 128;
  if (nkb <= 0 || T > max_t || dk % 16 != 0 || dk > GAM_REL_POS_MAX_DK || (cu != nullptr && klen == nullptr)) return -1;
  RelParams p;
  p.T = T;
  p.klen = klen;
  p.cu = cu;
  p.out = out;
  p.ld_out = d_model;
  p.dk = dk;
  p.pos_center = max_t - 1;
  p.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(dk));
  switch (dk / 16) {
    case 1: return launch_ks<1>(tmap_qkv, tmap_pos, p, nkb, B, H, s);
    case 2: return launch_ks<2>(tmap_qkv, tmap_pos, p, nkb, B, H, s);
    case 3: return launch_ks<3>(tmap_qkv, tmap_pos, p, nkb, B, H, s);
    default: return launch_ks<4>(tmap_qkv, tmap_pos, p, nkb, B, H, s);
  }
}

}  // namespace gam
