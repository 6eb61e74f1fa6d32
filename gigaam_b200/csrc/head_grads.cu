// Backward passes of the head kernels of heads.cu (CTC log-probs, RNN-T joint lattice, prediction LSTM), for training the
// heads on a frozen encoder.  All arithmetic is fp32 with expf / tanhf like the forward kernels.  No atomics: every sum
// runs in an order fixed by the sizes alone, so two calls on the same inputs give bit-identical gradients.
//   (1) softmax_grad_kernel: dlogit = G - exp(logp) * sum(G) per row (the backward of log_softmax).
//   (2) outer_sum_kernel: dW[N, K] = sum_r A[r, n] X(r, k) and db[n] = sum_r A[r, n], the weight gradient of every linear
//       map of the heads.  Rows are cut into S fixed slices; slice partials are added in slice order by outer_sum_reduce.
//       X(r, k) is read plainly, shifted by one step (the LSTM's previous hidden state) or rebuilt as the joint's
//       relu(E + P) hidden row, which is never stored.
//   (3) matmul_kernel: out[r, k] = sum_n A[r, n] W(n, k) (ascending n), optionally times [relu(E + P) > 0]: the input
//       gradients.
//   (4) segment_sum_kernel: sums of row groups in ascending order (the joint's sums over u and over t).
//   (5) lstm_bwd_step_kernel: one step of BPTT through lstm_step_kernel, one launch per step, last step first.
//   (6) class_gate_sum_kernel: the gate gradients of all steps whose input was class v, in row order.
#include <cmath>

#include "../../include/gigaam_b200.h"
#include "kernels.h"

namespace gam {
namespace {

// ------------------------------------------------------------------ (1) log_softmax backward
constexpr int kSgWarps = 8;

__global__ void __launch_bounds__(kSgWarps * 32) softmax_grad_kernel(const float* __restrict__ G, const float* __restrict__ logp,
                                                                      float* __restrict__ dl, int64_t rows, int V1) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * kSgWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* g = G + row * V1;
  const float* lp = logp + row * V1;
  float s = 0.f;
  for (int i = lane; i < V1; i += 32) s += g[i];
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  float* d = dl + row * V1;
  for (int i = lane; i < V1; i += 32) d[i] = g[i] - expf(lp[i]) * s;
}

// ------------------------------------------------------------------ X operands of the outer sums / masks
struct XPlain {   // X [rows, K]
  const float* X;
  int K;
  __device__ float operator()(int64_t r, int k) const { return X[r * K + k]; }
};
struct XShift {   // row r = (b, u) of U steps: X[r - 1] for u > 0, X0[b] (null: 0) for u = 0
  const float* X;
  const float* X0;
  int K, U;
  __device__ float operator()(int64_t r, int k) const {
    if (r % U != 0) return X[(r - 1) * K + k];
    return X0 != nullptr ? X0[(r / U) * K + k] : 0.f;
  }
};
struct XJoint {   // row r = (b, t, u): relu(E[b*T + t] + P[b*U + u]), NaN kept (rnnt_joint_kernel's hidden row)
  const float* E;
  const float* P;
  int K, T, U;
  __device__ float operator()(int64_t r, int k) const {
    const int64_t bt = r / U;
    const int64_t bu = bt / T * U + r % U;
    const float z = E[bt * K + k] + P[bu * K + k];
    return z < 0.f ? 0.f : z;
  }
};

// ------------------------------------------------------------------ (2) sum of outer products over rows
constexpr int kOT = 64, kOR = 16;   // 64 x 64 output tile, rows staged 16 at a time

// Column K of the tile (when db != null) is the all-ones column: its sums are db.  out: partials [S][N][Kc] when S > 1
// (Kc = K + 1 with db, else K), else written straight to dW / db.
template <class XOp>
__global__ void __launch_bounds__(256) outer_sum_kernel(const float* __restrict__ A, XOp xop, int64_t rows, int64_t chunk, int N,
                                                       int K, int Kc, float* part, float* dW, float* db) {
  __shared__ float a_s[kOR][kOT];
  __shared__ float x_s[kOR][kOT];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int k0 = blockIdx.x * kOT, n0 = blockIdx.y * kOT;
  const int64_t r_begin = static_cast<int64_t>(blockIdx.z) * chunk;
  const int64_t r_end = min(rows, r_begin + chunk);
  float acc[4][4] = {};
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kOR) {
    __syncthreads();
    for (int i = threadIdx.x; i < kOR * kOT; i += 256) {
      const int rr = i / kOT, c = i % kOT;
      const int64_t r = r0 + rr;
      const bool live = r < r_end;
      a_s[rr][c] = (live && n0 + c < N) ? A[r * N + n0 + c] : 0.f;
      const int k = k0 + c;
      x_s[rr][c] = (!live || k >= Kc) ? 0.f : (k == K ? 1.f : xop(r, k));
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kOR; ++rr) {
      float a[4], x[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = a_s[rr][ty * 4 + i]; x[i] = x_s[rr][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], x[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + ty * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx * 4 + j;
      if (k >= Kc) continue;
      if (part != nullptr)
        part[(static_cast<int64_t>(blockIdx.z) * N + n) * Kc + k] = acc[i][j];
      else if (k < K)
        dW[static_cast<int64_t>(n) * K + k] = acc[i][j];
      else
        db[n] = acc[i][j];
    }
  }
}

__global__ void outer_sum_reduce_kernel(const float* __restrict__ part, int S, int N, int K, int Kc, float* dW, float* db) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t NK = static_cast<int64_t>(N) * Kc;
  if (i >= NK) return;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += part[z * NK + i];
  const int n = static_cast<int>(i / Kc), k = static_cast<int>(i % Kc);
  if (k < K)
    dW[static_cast<int64_t>(n) * K + k] = s;
  else
    db[n] = s;
}

// ------------------------------------------------------------------ (3) out = A W (+ relu mask)
// W(n, k) = W[n * sn + k * sk]; mask (E != null): out[r, k] *= [relu(E + P)(r, k) > 0] (XJoint's row r)
__global__ void __launch_bounds__(256) matmul_kernel(const float* __restrict__ A, const float* __restrict__ W, int64_t sn, int64_t sk,
                                                     float* __restrict__ out, int64_t rows, int N, int K, XJoint mask) {
  __shared__ float a_s[kOR][kOT + 1];
  __shared__ float w_s[kOR][kOT];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kOT;
  const int k0 = blockIdx.y * kOT;
  float acc[4][4] = {};
  for (int nb = 0; nb < N; nb += kOR) {
    __syncthreads();
    for (int i = threadIdx.x; i < kOR * kOT; i += 256) {
      const int rr = i / kOR, nn = i % kOR;   // A: consecutive threads walk n of one row
      a_s[nn][rr] = (r0 + rr < rows && nb + nn < N) ? A[(r0 + rr) * N + nb + nn] : 0.f;
      const int n2 = i / kOT, c = i % kOT;
      w_s[n2][c] = (nb + n2 < N && k0 + c < K) ? W[(nb + n2) * sn + (k0 + c) * sk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int nn = 0; nn < kOR; ++nn) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = a_s[nn][ty * 4 + i]; w[i] = w_s[nn][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = r0 + ty * 4 + i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx * 4 + j;
      if (k >= K) continue;
      float v = acc[i][j];
      if (mask.E != nullptr && !(mask(r, k) > 0.f)) v = 0.f;
      out[r * K + k] = v;
    }
  }
}

// ------------------------------------------------------------------ (4) row-group sums
// out[g, k] = sum_{i < count} X[row(g, i), k], row(g, i) = (g / gi) * so + (g % gi) * si + i * step, i ascending
__global__ void segment_sum_kernel(const float* __restrict__ X, float* __restrict__ out, int64_t groups, int count, int K, int64_t gi,
                                   int64_t so, int64_t si, int64_t step) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= groups * K) return;
  const int64_t g = idx / K;
  const int k = static_cast<int>(idx % K);
  const float* p = X + ((g / gi) * so + (g % gi) * si) * K + k;
  float s = 0.f;
  for (int i = 0; i < count; ++i) s += p[i * step * K];
  out[idx] = s;
}

// ------------------------------------------------------------------ (5) BPTT step of the prediction LSTM
constexpr int kBPB = 4;          // utterances per block
constexpr int kBThreads = 64;    // hidden units per block

// Step u (>= 0) recomputes the gates of lstm_step_kernel from h_{u-1} (g[:, u-1] or h0) and the stored cells c_seq [U, B, H],
// takes dh_u = dG[b, u] + (u == U-1 ? dh1 : dgates_{u+1} W_hh) and the carried dc (dc_carry, initialised to dc1 by the
// caller), and writes dgates_u [B, U, 4H] (order i, f, g, o: gradients of the gate pre-activations) and dc_carry = dc_u * f_u.
// u = -1: dh0 = dgates_0 W_hh, dc0 = dc_carry.  An utterance whose ids leave [0, V1) gets NaN everywhere, as in the forward.
__global__ void __launch_bounds__(kBThreads) lstm_bwd_step_kernel(const int64_t* __restrict__ x, int U, int u, int V1,
                                                                  const float* __restrict__ emb_gates, const float* __restrict__ whh_t,
                                                                  const float* __restrict__ whh, const float* __restrict__ h0,
                                                                  const float* __restrict__ c0, const float* __restrict__ g,
                                                                  const float* __restrict__ c_seq, const float* __restrict__ dG,
                                                                  const float* __restrict__ dh1, float* __restrict__ dgates,
                                                                  float* __restrict__ dc_carry, float* __restrict__ dh0,
                                                                  float* __restrict__ dc0, int B, int H) {
  extern __shared__ float4 smem_f4[];
  float* h_s = reinterpret_cast<float*>(smem_f4);   // [kBPB][H]   h_{u-1}
  float* d_s = h_s + kBPB * H;                       // [kBPB][4H]  dgates_{u+1} (or dgates_0 when u = -1)
  __shared__ int bad_s[kBPB];
  const int H4 = 4 * H;
  const int j = blockIdx.x * kBThreads + threadIdx.x;
  const int b0 = blockIdx.y * kBPB;
  const int nb = min(kBPB, B - b0);
  if (threadIdx.x < kBPB) bad_s[threadIdx.x] = 0;
  __syncthreads();
  if (x != nullptr) {
    for (int i = threadIdx.x; i < nb * U; i += kBThreads) {
      const int64_t id = x[static_cast<int64_t>(b0) * U + i];
      if (id < 0 || id >= V1) bad_s[i / U] = 1;
    }
  }
  const int un = u + 1;   // the step whose gate gradients feed dh_u
  const bool have_next = u < 0 || un < U;
  for (int i = threadIdx.x; i < kBPB * H4; i += kBThreads) {
    const int bb = i / H4, q = i % H4;
    d_s[i] = (bb < nb && have_next) ? dgates[(static_cast<int64_t>(b0 + bb) * U + (u < 0 ? 0 : un)) * H4 + q] : 0.f;
  }
  if (u >= 0) {
    for (int i = threadIdx.x; i < kBPB * H; i += kBThreads) {
      const int bb = i / H, k = i % H;
      float v = 0.f;
      if (bb < nb) {
        if (u > 0)
          v = g[(static_cast<int64_t>(b0 + bb) * U + u - 1) * H + k];
        else if (h0 != nullptr)
          v = h0[static_cast<int64_t>(b0 + bb) * H + k];
      }
      h_s[i] = v;
    }
  }
  __syncthreads();
  if (j >= H) return;
  float dhr[kBPB];   // dgates_next W_hh, column j
#pragma unroll
  for (int bb = 0; bb < kBPB; ++bb) dhr[bb] = 0.f;
  if (have_next) {
    for (int q = 0; q < H4; ++q) {
      const float w = __ldg(whh + static_cast<size_t>(q) * H + j);
#pragma unroll
      for (int bb = 0; bb < kBPB; ++bb) dhr[bb] = fmaf(d_s[bb * H4 + q], w, dhr[bb]);
    }
  }
  if (u < 0) {
    for (int bb = 0; bb < nb; ++bb) {
      const int64_t o = static_cast<int64_t>(b0 + bb) * H + j;
      const float nan = __int_as_float(0x7fc00000);
      if (dh0 != nullptr) dh0[o] = bad_s[bb] ? nan : dhr[bb];
      if (dc0 != nullptr) dc0[o] = bad_s[bb] ? nan : dc_carry[o];
    }
    return;
  }
  float acc[4][kBPB];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int bb = 0; bb < kBPB; ++bb) acc[q][bb] = 0.f;
  for (int k = 0; k < H; ++k) {   // the forward's gate sums, in the forward's order
    const float* wr = whh_t + static_cast<size_t>(k) * H4 + j;
    const float w0 = __ldg(wr), w1 = __ldg(wr + H), w2 = __ldg(wr + 2 * H), w3 = __ldg(wr + 3 * H);
#pragma unroll
    for (int bb = 0; bb < kBPB; ++bb) {
      const float hv = h_s[bb * H + k];
      acc[0][bb] = fmaf(w0, hv, acc[0][bb]);
      acc[1][bb] = fmaf(w1, hv, acc[1][bb]);
      acc[2][bb] = fmaf(w2, hv, acc[2][bb]);
      acc[3][bb] = fmaf(w3, hv, acc[3][bb]);
    }
  }
  const int64_t BH = static_cast<int64_t>(B) * H;
#pragma unroll
  for (int bb = 0; bb < kBPB; ++bb) {
    if (bb >= nb) break;
    const int b = b0 + bb;
    const int64_t o = static_cast<int64_t>(b) * H + j;
    float* dgo = dgates + (static_cast<int64_t>(b) * U + u) * H4 + j;
    if (bad_s[bb]) {
      const float nan = __int_as_float(0x7fc00000);
      dgo[0] = dgo[H] = dgo[2 * H] = dgo[3 * H] = nan;
      dc_carry[o] = nan;
      continue;
    }
    const int64_t id = x != nullptr ? x[static_cast<int64_t>(b) * U + u] : V1 - 1;
    const float* eg = emb_gates + id * H4 + j;
    const float gi = acc[0][bb] + __ldg(eg), gf = acc[1][bb] + __ldg(eg + H);
    const float gg = acc[2][bb] + __ldg(eg + 2 * H), go = acc[3][bb] + __ldg(eg + 3 * H);
    const float si = 1.f / (1.f + expf(-gi)), sf = 1.f / (1.f + expf(-gf)), so = 1.f / (1.f + expf(-go));
    const float tg = tanhf(gg);
    const float cn = c_seq[u * BH + o];
    const float cp = u > 0 ? c_seq[(u - 1) * BH + o] : (c0 != nullptr ? c0[o] : 0.f);
    const float tc = tanhf(cn);
    const float dh = dG[(static_cast<int64_t>(b) * U + u) * H + j] + (un < U ? dhr[bb] : (dh1 != nullptr ? dh1[o] : 0.f));
    const float dc = dc_carry[o] + dh * so * (1.f - tc * tc);
    dgo[0] = dc * tg * si * (1.f - si);
    dgo[H] = dc * cp * sf * (1.f - sf);
    dgo[2 * H] = dc * si * (1.f - tg * tg);
    dgo[3 * H] = dh * tc * so * (1.f - so);
    dc_carry[o] = dc * sf;
  }
}

// ------------------------------------------------------------------ (6) gate gradients per input class
constexpr int kCThreads = 256;
constexpr int kCMaxPer = 16;   // 4H <= kCThreads * kCMaxPer

// out[v, :] = sum over rows r (ascending) with x[r] == v of dgates[r, :]; the blank row (padding_idx, zero embedding) is 0
__global__ void __launch_bounds__(kCThreads) class_gate_sum_kernel(const int64_t* __restrict__ x, int64_t rows,
                                                                   const float* __restrict__ dgates, int H4, int blank,
                                                                   float* __restrict__ out) {
  const int v = blockIdx.x;
  float acc[kCMaxPer];
#pragma unroll
  for (int i = 0; i < kCMaxPer; ++i) acc[i] = 0.f;
  if (v != blank) {
    for (int64_t r = 0; r < rows; ++r) {
      if (x[r] != v) continue;
      const float* d = dgates + r * H4;
#pragma unroll
      for (int i = 0; i < kCMaxPer; ++i) {
        const int q = threadIdx.x + i * kCThreads;
        if (q < H4) acc[i] += d[q];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < kCMaxPer; ++i) {
    const int q = threadIdx.x + i * kCThreads;
    if (q < H4) out[static_cast<int64_t>(v) * H4 + q] = acc[i];
  }
}

int outer_splits(int64_t rows, int N, int Kc) {
  const int64_t tiles = static_cast<int64_t>((N + kOT - 1) / kOT) * ((Kc + kOT - 1) / kOT);
  int64_t S = (264 + tiles - 1) / tiles;   // about two waves of CTAs on 132 SMs
  S = S < 1 ? 1 : (S > 64 ? 64 : S);
  const int64_t by_rows = (rows + 255) / 256;   // at least 256 rows per slice
  if (S > by_rows) S = by_rows < 1 ? 1 : by_rows;
  return static_cast<int>(S);
}

template <class XOp>
void outer_sum(const float* A, XOp xop, int64_t rows, int N, int K, float* dW, float* db, float* ws, cudaStream_t s) {
  const int Kc = K + (db != nullptr ? 1 : 0);
  const int S = outer_splits(rows, N, Kc);
  int64_t chunk = (rows + S - 1) / S;
  chunk = (chunk + kOR - 1) / kOR * kOR;
  dim3 grid((Kc + kOT - 1) / kOT, (N + kOT - 1) / kOT, S);
  outer_sum_kernel<<<grid, 256, 0, s>>>(A, xop, rows, chunk, N, K, Kc, S > 1 ? ws : nullptr, dW, db);
  if (S > 1) {
    const int64_t NK = static_cast<int64_t>(N) * Kc;
    outer_sum_reduce_kernel<<<static_cast<unsigned>((NK + 255) / 256), 256, 0, s>>>(ws, S, N, K, Kc, dW, db);
  }
}

}  // namespace

int64_t outer_sum_workspace_floats(int64_t rows, int N, int K, bool with_bias) {
  const int Kc = K + (with_bias ? 1 : 0);
  const int S = outer_splits(rows, N, Kc);
  return S > 1 ? static_cast<int64_t>(S) * N * Kc : 0;
}

void launch_softmax_grad(const float* G, const float* logp, float* dl, int64_t rows, int V1, cudaStream_t s) {
  if (rows <= 0) return;
  softmax_grad_kernel<<<static_cast<unsigned>((rows + kSgWarps - 1) / kSgWarps), kSgWarps * 32, 0, s>>>(G, logp, dl, rows, V1);
}

void launch_outer_sum(const float* A, const float* X, int64_t rows, int N, int K, float* dW, float* db, float* ws, cudaStream_t s) {
  outer_sum(A, XPlain{X, K}, rows, N, K, dW, db, ws, s);
}

void launch_outer_sum_shift(const float* A, const float* X, const float* X0, int U, int64_t rows, int N, int K, float* dW, float* db,
                            float* ws, cudaStream_t s) {
  outer_sum(A, XShift{X, X0, K, U}, rows, N, K, dW, db, ws, s);
}

void launch_outer_sum_joint(const float* A, const float* E, const float* P, int T, int U, int64_t rows, int N, int K, float* dW,
                            float* db, float* ws, cudaStream_t s) {
  outer_sum(A, XJoint{E, P, K, T, U}, rows, N, K, dW, db, ws, s);
}

void launch_outer_sum_reduce(const float* part, int S, int N, int K, int Kc, float* dW, float* db, cudaStream_t s) {
  const int64_t NK = static_cast<int64_t>(N) * Kc;
  outer_sum_reduce_kernel<<<static_cast<unsigned>((NK + 255) / 256), 256, 0, s>>>(part, S, N, K, Kc, dW, db);
}

void launch_head_matmul(const float* A, const float* W, int64_t sn, int64_t sk, float* out, int64_t rows, int N, int K,
                        const float* mask_E, const float* mask_P, int T, int U, cudaStream_t s) {
  if (rows <= 0) return;
  dim3 grid(static_cast<unsigned>((rows + kOT - 1) / kOT), (K + kOT - 1) / kOT);
  matmul_kernel<<<grid, 256, 0, s>>>(A, W, sn, sk, out, rows, N, K, XJoint{mask_E, mask_P, K, T, U});
}

void launch_segment_sum(const float* X, float* out, int64_t groups, int count, int K, int64_t gi, int64_t so, int64_t si, int64_t step,
                        cudaStream_t s) {
  const int64_t n = groups * K;
  if (n <= 0) return;
  segment_sum_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(X, out, groups, count, K, gi, so, si, step);
}

// lstm_bwd_step_kernel's dynamic shared memory: h_{u-1} and dgates of kBPB utterances, 5 H floats each, within the 48 KiB a
// launch gets without opting in
constexpr int kLstmBwdMaxHidden = 48 * 1024 / (kBPB * 5 * 4);
static_assert(kLstmBwdMaxHidden == GAM_PREDICT_BACKWARD_MAX_HIDDEN, "the header's pred_hidden limit of the predict backward");

int lstm_bwd_max_hidden() { return kLstmBwdMaxHidden; }

void launch_lstm_bwd_step(const int64_t* x, int U, int u, int V1, const float* emb_gates, const float* whh_t, const float* whh,
                          const float* h0, const float* c0, const float* g, const float* c_seq, const float* dG, const float* dh1,
                          float* dgates, float* dc_carry, float* dh0, float* dc0, int B, int H, cudaStream_t s) {
  dim3 grid((H + kBThreads - 1) / kBThreads, (B + kBPB - 1) / kBPB);
  lstm_bwd_step_kernel<<<grid, kBThreads, static_cast<size_t>(kBPB) * 5 * H * 4, s>>>(x, U, u, V1, emb_gates, whh_t, whh, h0, c0, g,
                                                                                     c_seq, dG, dh1, dgates, dc_carry, dh0, dc0, B, H);
}

int launch_class_gate_sum(const int64_t* x, int64_t rows, const float* dgates, int H4, int V1, int blank, float* out, cudaStream_t s) {
  if (H4 > kCThreads * kCMaxPer) return 1;
  class_gate_sum_kernel<<<V1, kCThreads, 0, s>>>(x, rows, dgates, H4, blank, out);
  return 0;
}

}  // namespace gam
