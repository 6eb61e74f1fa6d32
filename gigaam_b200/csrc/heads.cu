// Forward passes of the CTC and RNN-T heads as public calls (gigaam/decoder.py:18-21, 41-47, 85-102, 131-137): the
// posteriors and lattices callers feed to their own beam search, LM fusion, rescoring or alignment.  All arithmetic is
// fp32 on the CUDA cores, like the reference's heads (gigaam/__init__.py:188-189); every exp / log is expf / logf.
//   (1) ctc_log_probs_kernel: log_softmax(W enc + b) per frame.  Same tiling and the same ascending-k sums as
//       ctc_argmax_kernel (ctc.cu), so its pre-normalisation logits are bit-identical to the greedy path's.
//   (2) rnnt_joint_kernel: out[b,t,u,:] = log_softmax(W_o relu(E[b,t] + P[b,u]) + b_o) with E / P precomputed by
//       launch_sgemm_tn_bias / launch_sgemm_nn_bias.  The [rows, joint_hidden] hidden tile is built in shared memory and
//       never reaches HBM.
//   (3) lstm_step_kernel: one step of the 1-layer prediction LSTM over a batch, one launch per step.
//
// Normalising a row that spans several class tiles: both log-softmax kernels compute every logit ONCE, write it raw and
// keep a running (max, sum of exp) per row; when all class tiles are done the block subtracts max + log(sum) from the
// rows it just wrote (contiguous, coalesced, mostly still in L2).  The alternative, computing the logits twice (once for
// the statistics, once to write), doubles the GEMM, which is the dominant cost: at joint_hidden 320 a logit is 320 FMAs
// but the extra normalisation pass is one 4-byte read and write.
//
// Non-finite logits follow torch.log_softmax, as the greedy and scored paths of ctc.cu / rnnt_cluster.cu do: a -inf logit
// (a -inf bias bans a class) gives -inf at its class and leaves the rest of the row finite; a NaN or +inf logit, or a
// row whose logits are all -inf, gives a row of NaN.  The running log-sum-exp below skips -inf and lets NaN and +inf
// poison the sum; finite rows take the same branches as without the rule, so their bits do not depend on it.
#include <cmath>

#include "kernels.h"
#include "launch.cuh"

namespace gam {
namespace {

// running log-sum-exp: (m, s) = (max so far, sum of exp(v - m)).  m is never NaN; s is NaN once a NaN or a second +inf
// was pushed, and a +inf max turns s into NaN at the merge (exp(inf - inf)).
__device__ __forceinline__ void lse_push(float& m, float& s, float v) {
  if (v > m) {
    s = s * expf(m - v) + 1.f;
    m = v;
  } else if (v != -INFINITY) {   // -inf adds exp(-inf) = 0, but exp(-inf - -inf) = NaN while m is still -inf; NaN gets in
    s += expf(v - m);
  }
}

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  const float M = fmaxf(m, m2);
  if (M == -INFINITY) {   // neither side has a logit above -inf: their sums are 0, or NaN if a NaN was pushed
    s += s2;
    return;
  }
  s = s * expf(m - M) + s2 * expf(m2 - M);
  m = M;
}

// ------------------------------------------------------------------ (1) CTC log-probs
constexpr int kRows = 32;      // rows (frames) per block: thread = (row, class group), as in ctc_argmax_kernel
constexpr int kGroups = 4;
constexpr int kKC = 64;
constexpr int kCG = 9;
constexpr int kCT = kGroups * kCG;

__global__ void __launch_bounds__(kRows * kGroups) ctc_log_probs_kernel(const float* __restrict__ enc, const float* __restrict__ W,
                                                                        const float* __restrict__ bias, float* __restrict__ out,
                                                                        int R, int D, int V1) {
  __shared__ float e_s[kKC][kRows + 1];
  __shared__ float w_s[kCT][kKC];
  __shared__ float red_m[kGroups][kRows];
  __shared__ float red_s[kGroups][kRows];
  __shared__ float lse_s[kRows];
  const int r = threadIdx.x & 31, cg = threadIdx.x >> 5;
  const int row0 = blockIdx.x * kRows;
  const bool live = row0 + r < R;
  float* orow = out + static_cast<size_t>(row0 + r) * V1;
  float m = -INFINITY, sum = 0.f;
  for (int c0 = 0; c0 < V1; c0 += kCT) {
    float acc[kCG];
#pragma unroll
    for (int c = 0; c < kCG; ++c) acc[c] = 0.f;
    for (int k0 = 0; k0 < D; k0 += kKC) {
      __syncthreads();
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
        lse_push(m, sum, v);
        if (live) orow[cls] = v;
      }
    }
  }
  red_m[cg][r] = m;
  red_s[cg][r] = sum;
  __syncthreads();
  if (cg == 0) {
#pragma unroll
    for (int g = 1; g < kGroups; ++g) lse_merge(m, sum, red_m[g][r], red_s[g][r]);
    lse_s[r] = m + logf(sum);
  }
  __syncthreads();   // also orders the raw-logit stores above before the re-reads below (block scope)
  const int n = min(kRows, R - row0) * V1;
  float* base = out + static_cast<size_t>(row0) * V1;
  for (int i = threadIdx.x; i < n; i += kRows * kGroups) base[i] -= lse_s[i / V1];
}

// ------------------------------------------------------------------ (2) RNN-T joint lattice
constexpr int kJBM = 64, kJBN = 64, kJBK = 16;   // rows x classes per block tile, K chunk of the W_o stream
constexpr int kJLd = kJBM + 4;                     // A_s / W_s row pitch (floats)
constexpr int kJThreads = 256;                     // 16 x 16 threads, 4 x 4 outputs each

__host__ __device__ constexpr int joint_kpad(int J) { return (J + kJBK - 1) / kJBK * kJBK; }
__host__ __device__ constexpr size_t joint_smem_bytes(int J) { return (static_cast<size_t>(joint_kpad(J)) + kJBK) * kJLd * 4; }

// E [B*T, J], P [B*U, J] (biases included), W_o [V1, J], b_o [V1] -> out [B, T, U, V1], row (b, t, u) = (b*T + t)*U + u.
// kGather (gam_rnnt_align_scores): the same rows, tiles and running statistics, but of each row only the blank logit and
// the logit of the row's next label are kept: U = U_y + 1 lattice columns, targets [B, U_y] i32, and
//   blank_out[row] = log_softmax(row)[V1 - 1],  label_out[row] = log_softmax(row)[targets[b, u]] for u < U_y
// (NaN for an id outside [0, V1 - 1), -inf at u = U_y).  Each is the same fp32 subtraction as the lattice's, so it is
// bit-identical to the matching lattice entry.  out is unused and no [V1] row is stored.  kLse (gam_rnnt_loss, gather mode
// only): lse_out[row] also receives the row's log-sum-exp, the value both gathered entries subtract.
template <bool kGather, bool kLse = false>
__global__ void __launch_bounds__(kJThreads) rnnt_joint_kernel(const float* __restrict__ E, const float* __restrict__ P,
                                                               const float* __restrict__ Wo, const float* __restrict__ bo,
                                                               float* __restrict__ out, int T, int U, int J, int V1,
                                                               int64_t rows, const int* __restrict__ targets,
                                                               float* __restrict__ blank_out, float* __restrict__ label_out,
                                                               float* __restrict__ lse_out) {
  extern __shared__ float4 smem_f4[];
  float* A_s = reinterpret_cast<float*>(smem_f4);   // [Jp][kJLd]: relu(E + P) of the block's rows, k-major
  const int Jp = joint_kpad(J);
  float* W_s = A_s + static_cast<size_t>(Jp) * kJLd;   // [kJBK][kJLd]: W_o chunk, k-major
  __shared__ float lse_s[kJBM];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * kJBM;
  // kGather: the kept raw logits and the label id of each row of the block (-1: none, -2: id out of range), behind W_s
  float* blank_s = W_s + kJBK * kJLd;
  float* label_s = blank_s + kJBM;
  int* y_s = reinterpret_cast<int*>(label_s + kJBM);
  if constexpr (kGather) {
    if (tid < kJBM) {
      const int64_t row = row0 + tid;
      int y = -1;
      if (row < rows && row % U < U - 1) {
        y = targets[row / U / T * (U - 1) + row % U];
        if (y < 0 || y >= V1 - 1) y = -2;
      }
      y_s[tid] = y;   // read after the main loop's barriers
    }
  }

  const int J4 = J / 4;
  for (int i = tid; i < kJBM * J4; i += kJThreads) {
    const int m = i / J4, k4 = (i % J4) * 4;
    const int64_t row = row0 + m;
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < rows) {
      const int64_t bt = row / U;
      const int64_t bu = bt / T * U + row % U;
      const float4 e = *reinterpret_cast<const float4*>(E + bt * J + k4);
      const float4 p = *reinterpret_cast<const float4*>(P + bu * J + k4);
      // relu that keeps NaN, as torch.relu (fmaxf(NaN, 0) = 0 would give finite log-probs where the reference has NaN)
      const float z0 = e.x + p.x, z1 = e.y + p.y, z2 = e.z + p.z, z3 = e.w + p.w;
      z = make_float4(z0 < 0.f ? 0.f : z0, z1 < 0.f ? 0.f : z1, z2 < 0.f ? 0.f : z2, z3 < 0.f ? 0.f : z3);
    }
    A_s[(k4 + 0) * kJLd + m] = z.x;
    A_s[(k4 + 1) * kJLd + m] = z.y;
    A_s[(k4 + 2) * kJLd + m] = z.z;
    A_s[(k4 + 3) * kJLd + m] = z.w;
  }
  for (int i = tid; i < (Jp - J) * kJBM; i += kJThreads) A_s[(J + i / kJBM) * kJLd + i % kJBM] = 0.f;

  float rm[4], rs[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { rm[i] = -INFINITY; rs[i] = 0.f; }
  for (int n0 = 0; n0 < V1; n0 += kJBN) {
    float acc[4][4] = {};
    for (int k0 = 0; k0 < Jp; k0 += kJBK) {
      __syncthreads();   // A_s complete (first pass); previous W_s chunk consumed
      {
        const int r = tid / 4, k4 = (tid % 4) * 4;
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n0 + r < V1 && k0 + k4 < J) w = __ldg(reinterpret_cast<const float4*>(Wo + static_cast<size_t>(n0 + r) * J + k0 + k4));
        W_s[(k4 + 0) * kJLd + r] = w.x;
        W_s[(k4 + 1) * kJLd + r] = w.y;
        W_s[(k4 + 2) * kJLd + r] = w.z;
        W_s[(k4 + 3) * kJLd + r] = w.w;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kJBK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(A_s + (k0 + k) * kJLd + ty * 4);
        const float4 w = *reinterpret_cast<const float4*>(W_s + k * kJLd + tx * 4);
        const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t row = row0 + ty * 4 + i;
      float* orow = out + row * V1;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        if (n < V1) {
          const float v = acc[i][j] + __ldg(bo + n);
          lse_push(rm[i], rs[i], v);
          if constexpr (kGather) {
            if (n == V1 - 1) blank_s[ty * 4 + i] = v;
            if (n == y_s[ty * 4 + i]) label_s[ty * 4 + i] = v;
          } else {
            if (row < rows) orow[n] = v;
          }
        }
      }
    }
  }
  // the 16 threads of one row group are 16 consecutive lanes: merge their statistics with xor shuffles inside the half-warp
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, rm[i], off);
      const float s2 = __shfl_xor_sync(0xffffffffu, rs[i], off);
      lse_merge(rm[i], rs[i], m2, s2);
    }
    if (tx == 0) lse_s[ty * 4 + i] = rm[i] + logf(rs[i]);
  }
  __syncthreads();
  if constexpr (kGather) {
    const int64_t row = row0 + tid;
    if (tid < kJBM && row < rows) {
      blank_out[row] = blank_s[tid] - lse_s[tid];
      const int y = y_s[tid];
      label_out[row] = y >= 0 ? label_s[tid] - lse_s[tid] : (y == -1 ? -INFINITY : __int_as_float(0x7fc00000));
      if constexpr (kLse) lse_out[row] = lse_s[tid];
    }
    return;
  }
  const int64_t left = rows - row0;
  const int n = static_cast<int>(left < kJBM ? left : kJBM) * V1;
  float* base = out + row0 * V1;
  for (int i = tid; i < n; i += kJThreads) base[i] -= lse_s[i / V1];
}

// ------------------------------------------------------------------ (3) prediction LSTM step
constexpr int kPB = 8;          // utterances per block
constexpr int kPThreads = 64;   // hidden units per block (one thread per unit, all four gates)

// gates = emb_gates[id] + h W_hh^T (emb_gates = embed W_ih^T + b_ih + b_hh), order i, f, g, o (gigaam/decoder.py:82).
// x: i64 [B, U] or null (every step reads the zero-embedding row `blank`).  h_in: [B] rows of pitch h_pitch, or null = 0.
// c_in: [B, H] or null = 0; may alias c_out (each thread reads its own element before writing it).  Writes
// g[(b*U + u)*H + j] = h', c_out[b*H + j] = c', and h_out[b*H + j] = h' when h_out != null.  An utterance whose ids leave
// [0, V1) gets NaN in everything it writes, and no table row is read for it.
__global__ void __launch_bounds__(kPThreads) lstm_step_kernel(const int64_t* __restrict__ x, int U, int u, int V1,
                                                              const float* __restrict__ emb_gates, const float* __restrict__ whh_t,
                                                              const float* __restrict__ h_in, int64_t h_pitch, const float* c_in,
                                                              float* __restrict__ g, float* __restrict__ h_out, float* c_out,
                                                              int B, int H) {
  extern __shared__ float4 smem_f4[];
  float* h_s = reinterpret_cast<float*>(smem_f4);   // [kPB][H]
  __shared__ int bad_s[kPB];
  const int j = blockIdx.x * kPThreads + threadIdx.x;
  const int b0 = blockIdx.y * kPB;
  const int nb = min(kPB, B - b0);
  if (threadIdx.x < kPB) bad_s[threadIdx.x] = 0;
  __syncthreads();
  if (x != nullptr) {
    for (int i = threadIdx.x; i < nb * U; i += kPThreads) {
      const int64_t id = x[static_cast<int64_t>(b0) * U + i];
      if (id < 0 || id >= V1) bad_s[i / U] = 1;
    }
  }
  for (int i = threadIdx.x; i < kPB * H; i += kPThreads) {
    const int bb = i / H, k = i % H;
    h_s[i] = (bb < nb && h_in != nullptr) ? h_in[static_cast<int64_t>(b0 + bb) * h_pitch + k] : 0.f;
  }
  __syncthreads();
  if (j >= H) return;
  const int H4 = 4 * H;
  float acc[4][kPB];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int bb = 0; bb < kPB; ++bb) acc[q][bb] = 0.f;
  for (int k = 0; k < H; ++k) {
    const float* wr = whh_t + static_cast<size_t>(k) * H4 + j;
    const float w0 = __ldg(wr), w1 = __ldg(wr + H), w2 = __ldg(wr + 2 * H), w3 = __ldg(wr + 3 * H);
#pragma unroll
    for (int bb = 0; bb < kPB; ++bb) {
      const float hv = h_s[bb * H + k];
      acc[0][bb] = fmaf(w0, hv, acc[0][bb]);
      acc[1][bb] = fmaf(w1, hv, acc[1][bb]);
      acc[2][bb] = fmaf(w2, hv, acc[2][bb]);
      acc[3][bb] = fmaf(w3, hv, acc[3][bb]);
    }
  }
#pragma unroll
  for (int bb = 0; bb < kPB; ++bb) {
    if (bb >= nb) break;
    const int b = b0 + bb;
    float hn, cn;
    if (bad_s[bb]) {
      hn = cn = __int_as_float(0x7fc00000);
    } else {
      const int64_t id = x != nullptr ? x[static_cast<int64_t>(b) * U + u] : V1 - 1;
      const float* eg = emb_gates + id * H4 + j;
      const float gi = acc[0][bb] + __ldg(eg), gf = acc[1][bb] + __ldg(eg + H);
      const float gg = acc[2][bb] + __ldg(eg + 2 * H), go = acc[3][bb] + __ldg(eg + 3 * H);
      const float cp = c_in != nullptr ? c_in[static_cast<int64_t>(b) * H + j] : 0.f;
      const float si = 1.f / (1.f + expf(-gi)), sf = 1.f / (1.f + expf(-gf)), so = 1.f / (1.f + expf(-go));
      cn = sf * cp + si * tanhf(gg);
      hn = so * tanhf(cn);
    }
    g[(static_cast<int64_t>(b) * U + u) * H + j] = hn;
    c_out[static_cast<int64_t>(b) * H + j] = cn;
    if (h_out != nullptr) h_out[static_cast<int64_t>(b) * H + j] = hn;
  }
}

}  // namespace

void launch_ctc_log_probs(const float* enc, const float* W, const float* bias, float* out, int R, int D, int V1, cudaStream_t s) {
  ctc_log_probs_kernel<<<(R + kRows - 1) / kRows, kRows * kGroups, 0, s>>>(enc, W, bias, out, R, D, V1);
}

int rnnt_joint_max_hidden() {
  int J = kJBK;
  while (joint_smem_bytes(J + kJBK) <= kJointMaxSmem) J += kJBK;
  return J;
}

int launch_rnnt_joint(const float* E, const float* P, const float* Wo, const float* bo, float* out, int B, int T, int U, int J,
                      int V1, cudaStream_t s) {
  static PerDeviceOnce attr_once;
  if (J % 4 != 0 || J > rnnt_joint_max_hidden()) return 1;
  if (attr_once.first() &&
      cudaFuncSetAttribute(rnnt_joint_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kJointMaxSmem)) !=
          cudaSuccess)
    return -1;
  const int64_t rows = static_cast<int64_t>(B) * T * U;
  const int64_t blocks = (rows + kJBM - 1) / kJBM;
  if (blocks > 0x7fffffff) return 1;
  rnnt_joint_kernel<false><<<static_cast<unsigned>(blocks), kJThreads, joint_smem_bytes(J), s>>>(E, P, Wo, bo, out, T, U, J, V1, rows,
                                                                                                  nullptr, nullptr, nullptr, nullptr);
  return 0;
}

int launch_rnnt_joint_gather(const float* E, const float* P, const float* Wo, const float* bo, const int* targets, float* blank,
                             float* label, float* lse, int B, int T, int U1, int J, int V1, cudaStream_t s) {
  static PerDeviceOnce attr_once;
  constexpr size_t kExtra = 3 * kJBM * 4;   // blank_s, label_s, y_s
  if (J % 4 != 0 || J > rnnt_joint_max_hidden()) return 1;
  if (attr_once.first() &&
      (cudaFuncSetAttribute(rnnt_joint_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            static_cast<int>(kJointMaxSmem + kExtra)) != cudaSuccess ||
       cudaFuncSetAttribute(rnnt_joint_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            static_cast<int>(kJointMaxSmem + kExtra)) != cudaSuccess))
    return -1;
  const int64_t rows = static_cast<int64_t>(B) * T * U1;
  const int64_t blocks = (rows + kJBM - 1) / kJBM;
  if (blocks > 0x7fffffff) return 1;
  if (lse != nullptr)
    rnnt_joint_kernel<true, true><<<static_cast<unsigned>(blocks), kJThreads, joint_smem_bytes(J) + kExtra, s>>>(
        E, P, Wo, bo, nullptr, T, U1, J, V1, rows, targets, blank, label, lse);
  else
    rnnt_joint_kernel<true><<<static_cast<unsigned>(blocks), kJThreads, joint_smem_bytes(J) + kExtra, s>>>(
        E, P, Wo, bo, nullptr, T, U1, J, V1, rows, targets, blank, label, nullptr);
  return 0;
}

void launch_lstm_step(const int64_t* x, int U, int u, int V1, const float* emb_gates, const float* whh_t, const float* h_in,
                      int64_t h_pitch, const float* c_in, float* g, float* h_out, float* c_out, int B, int H, cudaStream_t s) {
  dim3 grid((H + kPThreads - 1) / kPThreads, (B + kPB - 1) / kPB);
  lstm_step_kernel<<<grid, kPThreads, static_cast<size_t>(kPB) * H * 4, s>>>(x, U, u, V1, emb_gates, whh_t, h_in, h_pitch, c_in, g,
                                                                             h_out, c_out, B, H);
}

}  // namespace gam
