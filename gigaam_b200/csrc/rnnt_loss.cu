// Fused RNN-T loss and its gradient (include/gigaam_b200.h, gam_rnnt_loss / gam_rnnt_loss_backward, has the definitions).
// Nothing of size [nodes, V+1] or [nodes, joint_hidden] ever reaches global memory: the forward keeps three floats per
// lattice node (lse, e_blank, e_label) and the backward rebuilds the joint's hidden rows and logits tile by tile.
//   (1) rnnt_loss_alpha_beta_kernel: one CTA per utterance.  The forward walk over anti-diagonals is rnnt_align_kernel's
//       (same operands, same lse2, same order), so the loss is -log_likelihood of gam_rnnt_align bit for bit; alpha of every
//       node goes to scratch.  The backward walk keeps beta of two diagonals in shared memory and writes each node's edge
//       occupancies e_blank / e_label.
//   (2) rnnt_loss_node_grad_kernel: a CTA owns a strip of lattice columns (tU of them) of one utterance and a range of
//       frames, and walks 64-node tiles of tT x tU nodes down it.  Per tile: relu(E + P) in shared memory, then per class
//       tile of 64 the logits (rnnt_joint_kernel's sums), dz, and dhid += dz W_o in registers.  Masked by [E + P > 0],
//       dhid is summed over the tile's columns into a dE partial per (strip, frame) and over its frames into the strip's
//       dP accumulator, written once per CTA as a partial per (frame range, column).
//   (3) rnnt_loss_class_grad_kernel: a CTA owns a class tile and a slice of the flattened nodes, recomputes the logits of
//       its classes and accumulates dW_o^T (and db_o) in registers; slice partials are added in slice order by
//       outer_sum_reduce_kernel (head_grads.cu).
// All fp32 with expf / logf, no atomics, every sum in an order fixed by the sizes: repeated calls give the same bits.
#include <cmath>

#include "../../include/gigaam_b200.h"
#include "kernels.h"
#include "launch.cuh"

namespace gam {
namespace {

__device__ __forceinline__ float lse2(float a, float b) {   // align.cu's
  const float m = fmaxf(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log1pf(expf(fminf(a, b) - m));
}

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

// ------------------------------------------------------------------ (1) alpha / beta
// blank / label / alpha / e_blank / e_label: [B, T, U + 1].  Nodes outside utterance b's lattice get e = 0.
__global__ void rnnt_loss_alpha_beta_kernel(const float* __restrict__ blank, const float* __restrict__ label,
                                            const int* __restrict__ enc_len, const int* __restrict__ target_len, int T, int U,
                                            float* __restrict__ alpha, float* __restrict__ e_blank, float* __restrict__ e_label,
                                            float* __restrict__ loss) {
  extern __shared__ float4 smem_f4[];
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int U1 = U + 1;
  const int Tb = min(max(enc_len[b], 0), T), Ub = min(max(target_len[b], 0), U);
  float* fa = reinterpret_cast<float*>(smem_f4);   // [U1] per diagonal, indexed by u
  float* fb = fa + U1;
  __shared__ float ll_s;
  const int64_t off = static_cast<int64_t>(b) * T * U1;
  const float* bl = blank + off;
  const float* lb = label + off;
  float* al = alpha + off;
  float* eb = e_blank + off;
  float* el = e_label + off;
  for (int64_t i = tid; i < static_cast<int64_t>(T) * U1; i += nt) {
    if (i / U1 >= Tb || i % U1 > Ub) eb[i] = el[i] = 0.f;
  }
  int nan = 0;
  const int D = Tb - 1 + Ub;
  if (Tb > 0) {
    if (tid == 0) fa[0] = al[0] = 0.f;
    for (int d = 1; d <= D; ++d) {
      __syncthreads();   // diagonal d - 1 complete
      const int lo = max(0, d - (Tb - 1)), hi = min(Ub, d);
      for (int u = lo + tid; u <= hi; u += nt) {
        const int t = d - u;
        float fbk = -INFINITY, flk = -INFINITY;
        if (t > 0) {
          const float x = bl[static_cast<int64_t>(t - 1) * U1 + u];
          nan |= isnan(x);
          fbk = fa[u] + x;
        }
        if (u > 0) {
          const float x = lb[static_cast<int64_t>(t) * U1 + u - 1];
          nan |= isnan(x);
          flk = fa[u - 1] + x;
        }
        const float v = lse2(fbk, flk);
        fb[u] = v;
        al[static_cast<int64_t>(t) * U1 + u] = v;
      }
      float* tmp = fa; fa = fb; fb = tmp;
    }
  }
  float x_end = 0.f;
  if (tid == 0 && Tb > 0) {
    x_end = bl[static_cast<int64_t>(Tb - 1) * U1 + Ub];
    nan |= isnan(x_end);
  }
  nan = __syncthreads_or(nan);
  if (tid == 0) {
    float fwd = Tb > 0 ? fa[Ub] + x_end : -INFINITY;
    if (nan) fwd = qnan();
    loss[b] = -fwd;
    ll_s = fwd;
  }
  __syncthreads();
  const float ll = ll_s;
  const bool none = ll == -INFINITY;   // no path: the utterance contributes no gradient
  // beta(t, u) = lse2(blank(t, u) + beta(t + 1, u), label(t, u) + beta(t, u + 1)), beta(T_b, U_b) = 0 closing the lattice.
  // fa holds diagonal d + 1 (indexed by u), fb receives diagonal d.
  for (int d = D; d >= 0; --d) {
    __syncthreads();
    const int lo = max(0, d - (Tb - 1)), hi = min(Ub, d);
    for (int u = lo + tid; u <= hi; u += nt) {
      const int t = d - u;
      const int64_t n = static_cast<int64_t>(t) * U1 + u;
      const float a = al[n], xb = bl[n];
      const float bb = t + 1 < Tb ? fa[u] : (u == Ub ? 0.f : -INFINITY);
      float lab = -INFINITY, gl = 0.f;
      if (u < Ub) {
        const float xl = lb[n], bu = fa[u + 1];
        lab = xl + bu;
        gl = expf(a + xl + bu - ll);
      }
      fb[u] = lse2(xb + bb, lab);
      const float gb = expf(a + xb + bb - ll);
      eb[n] = none ? 0.f : gb;
      el[n] = none ? 0.f : gl;
    }
    float* tmp = fa; fa = fb; fb = tmp;
  }
}

// ------------------------------------------------------------------ shared pieces of (2) and (3)
constexpr int kLM = 64, kLN = 64, kLK = 16;   // nodes x classes per tile, K chunk of the W_o stream (rnnt_joint_kernel's)
constexpr int kLLd = kLM + 4;                  // row pitch of the k-major tiles (floats)
constexpr int kLThreads = 256;                 // 16 x 16 threads, 4 x 4 logits each
constexpr int kLMaxNC = 6;                     // 64-wide column chunks of joint_hidden held in registers: J <= 384

__host__ __device__ constexpr int loss_kpad(int J) { return (J + kLK - 1) / kLK * kLK; }
__host__ __device__ constexpr int loss_nc(int J) { return (J + 63) / 64; }

// Per-row operands of a tile, in shared memory.  e_row < 0 marks a node outside its utterance's lattice.
struct RowInfo {
  int64_t e_row[kLM], p_row[kLM];
  float lse[kLM], eb[kLM], el[kLM], g[kLM];
  int y[kLM];
};

// Row m of the tile is node (b, t, u); fills info (tid < kLM) for it.
__device__ __forceinline__ void stage_row(RowInfo& ri, int m, bool in_range, int b, int t, int u, int T, int U, const int* enc_len,
                                          const int* target_len, const int* targets, const float* lse, const float* e_blank,
                                          const float* e_label, const float* grad) {
  const int U1 = U + 1;
  bool live = in_range;
  int Ub = 0;
  if (live) {
    const int Tb = min(max(enc_len[b], 0), T);
    Ub = min(max(target_len[b], 0), U);
    live = t < Tb && u <= Ub;
  }
  ri.e_row[m] = live ? static_cast<int64_t>(b) * T + t : -1;
  ri.p_row[m] = live ? static_cast<int64_t>(b) * U1 + u : -1;
  if (live) {
    const int64_t n = (static_cast<int64_t>(b) * T + t) * U1 + u;
    ri.lse[m] = lse[n];
    ri.eb[m] = e_blank[n];
    ri.el[m] = e_label[n];
    ri.g[m] = grad[b];
    ri.y[m] = u < Ub ? targets[static_cast<int64_t>(b) * U + u] : -1;
  }
}

// A_s [rows][kLLd] (k-major) = relu(E + P) of the tile's live rows (NaN kept, as rnnt_joint_kernel), 0 for dead rows and
// for k in [J, rows)
__device__ __forceinline__ void stage_hidden(float* A_s, int rows, const RowInfo& ri, const float* E, const float* P, int J, int tid) {
  const int J4 = J / 4;
  for (int i = tid; i < kLM * J4; i += kLThreads) {
    const int m = i / J4, k4 = (i % J4) * 4;
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ri.e_row[m] >= 0) {
      const float4 e = *reinterpret_cast<const float4*>(E + ri.e_row[m] * J + k4);
      const float4 p = *reinterpret_cast<const float4*>(P + ri.p_row[m] * J + k4);
      const float z0 = e.x + p.x, z1 = e.y + p.y, z2 = e.z + p.z, z3 = e.w + p.w;
      z = make_float4(z0 < 0.f ? 0.f : z0, z1 < 0.f ? 0.f : z1, z2 < 0.f ? 0.f : z2, z3 < 0.f ? 0.f : z3);
    }
    A_s[(k4 + 0) * kLLd + m] = z.x;
    A_s[(k4 + 1) * kLLd + m] = z.y;
    A_s[(k4 + 2) * kLLd + m] = z.z;
    A_s[(k4 + 3) * kLLd + m] = z.w;
  }
  for (int i = tid; i < (rows - J) * kLM; i += kLThreads) A_s[(J + i / kLM) * kLLd + i % kLM] = 0.f;
}

// logits of rows ty*4 + i, classes n0 + tx*4 + j without the bias: rnnt_joint_kernel's sums, in its order
__device__ __forceinline__ void logit_tile(const float* A_s, float* W_s, const float* __restrict__ Wo, int n0, int J, int V1, int tid,
                                           float acc[4][4]) {
  const int tx = tid % 16, ty = tid / 16;
  const int Jp = loss_kpad(J);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < Jp; k0 += kLK) {
    __syncthreads();   // A_s complete (first chunk); previous W_s chunk consumed
    {
      const int r = tid / 4, k4 = (tid % 4) * 4;
      float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n0 + r < V1 && k0 + k4 < J) w = __ldg(reinterpret_cast<const float4*>(Wo + static_cast<size_t>(n0 + r) * J + k0 + k4));
      W_s[(k4 + 0) * kLLd + r] = w.x;
      W_s[(k4 + 1) * kLLd + r] = w.y;
      W_s[(k4 + 2) * kLLd + r] = w.z;
      W_s[(k4 + 3) * kLLd + r] = w.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kLK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(A_s + (k0 + k) * kLLd + ty * 4);
      const float4 w = *reinterpret_cast<const float4*>(W_s + k * kLLd + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
  }
}

// dz of row m, class n from its logit without bias: g (exp(z - lse) gamma - [n = blank] e_blank - [n = y] e_label), 0 for a dead
// row or a class past V1
__device__ __forceinline__ float dz_of(const RowInfo& ri, int m, int n, float acc, const float* __restrict__ bo, int V1) {
  if (ri.e_row[m] < 0 || n >= V1) return 0.f;
  const float z = acc + __ldg(bo + n);
  const float eb = ri.eb[m], el = ri.el[m];
  float d = expf(z - ri.lse[m]) * (eb + el);
  if (n == V1 - 1) d -= eb;
  if (n == ri.y[m]) d -= el;
  return ri.g[m] * d;
}

// ------------------------------------------------------------------ (2) node-major: dE / dP partials
// grid (NS strips, ST frame ranges, B).  Strip s: columns [s tU, (s + 1) tU); range r: frame tiles [r chunk, (r + 1) chunk) of
// tT frames.  dE_part [NS][B*T][J], dP_part [ST][B*U1][J].
template <int NC>
__global__ void __launch_bounds__(kLThreads) rnnt_loss_node_grad_kernel(
    const float* __restrict__ E, const float* __restrict__ P, const float* __restrict__ Wo, const float* __restrict__ bo,
    const int* __restrict__ targets, const int* __restrict__ enc_len, const int* __restrict__ target_len, const float* __restrict__ lse,
    const float* __restrict__ e_blank, const float* __restrict__ e_label, const float* __restrict__ grad, int B, int T, int U, int J,
    int V1, int tU, int chunk, float* __restrict__ dE_part, float* __restrict__ dP_part) {
  extern __shared__ float4 smem_f4[];
  const int Jp = loss_kpad(J), JW = NC * 64;
  float* A_s = reinterpret_cast<float*>(smem_f4);   // [Jp][kLLd] relu(E + P), then dhid
  float* W_s = A_s + Jp * kLLd;                      // [kLK][kLLd] W_o chunk of the logits
  float* dz_s = W_s + kLK * kLLd;                    // [kLN][kLLd] dz, class-major
  float* Wd_s = dz_s + kLN * kLLd;                   // [kLK][JW] W_o rows of the dhid product
  float* dP_s = Wd_s + kLK * JW;                     // [tU][J] the strip's dP accumulator
  __shared__ RowInfo ri;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int U1 = U + 1, tT = kLM / tU;
  const int strip = blockIdx.x, range = blockIdx.y, b = blockIdx.z;
  const int u0 = strip * tU;
  const int Tb = min(max(enc_len[b], 0), T), Ub = min(max(target_len[b], 0), U);
  for (int i = tid; i < tU * J; i += kLThreads) dP_s[i] = 0.f;
  const int n_tiles = (T + tT - 1) / tT;
  const int tile_end = min(n_tiles, (range + 1) * chunk);
  for (int tile = range * chunk; tile < tile_end; ++tile) {
    const int t0 = tile * tT;
    const bool live = t0 < Tb && u0 <= Ub;
    if (!live) {   // no node of the tile is in the lattice: its dE partials are 0 and dP is unchanged
      for (int i = tid; i < tT * J; i += kLThreads) {
        const int t = t0 + i / J;
        if (t < T) dE_part[((static_cast<int64_t>(strip) * B + b) * T + t) * J + i % J] = 0.f;
      }
      continue;
    }
    __syncthreads();   // the previous tile's sums are done with A_s and ri
    if (tid < kLM) {
      const int t = t0 + tid / tU, u = u0 + tid % tU;
      stage_row(ri, tid, t < T && u < U1, b, t, u, T, U, enc_len, target_len, targets, lse, e_blank, e_label, grad);
    }
    __syncthreads();
    stage_hidden(A_s, Jp, ri, E, P, J, tid);
    float dh[4][NC * 4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int c = 0; c < NC * 4; ++c) dh[i][c] = 0.f;
    for (int n0 = 0; n0 < V1; n0 += kLN) {
      float acc[4][4];
      logit_tile(A_s, W_s, Wo, n0, J, V1, tid, acc);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dz_s[(tx * 4 + j) * kLLd + ty * 4 + i] = dz_of(ri, ty * 4 + i, n0 + tx * 4 + j, acc[i][j], bo, V1);
      for (int kc = 0; kc < kLN; kc += kLK) {
        __syncthreads();   // dz_s written (first chunk); previous Wd_s chunk consumed
        for (int i = tid; i < kLK * (JW / 4); i += kLThreads) {
          const int r = i / (JW / 4), k4 = (i % (JW / 4)) * 4;
          const int n = n0 + kc + r;
          float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
          if (n < V1 && k4 < J) w = __ldg(reinterpret_cast<const float4*>(Wo + static_cast<size_t>(n) * J + k4));
          *reinterpret_cast<float4*>(Wd_s + r * JW + k4) = w;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kLK; ++k) {
          const float4 a = *reinterpret_cast<const float4*>(dz_s + (kc + k) * kLLd + ty * 4);
          const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const float4 w = *reinterpret_cast<const float4*>(Wd_s + k * JW + c * 64 + tx * 4);
            const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) dh[i][c * 4 + j] = fmaf(av[i], wv[j], dh[i][c * 4 + j]);
          }
        }
      }
    }
    __syncthreads();   // every thread is done reading A_s as the hidden rows
    // dhid = (dz W_o) * [hid > 0], in place of the hidden rows (each thread rewrites only its own elements)
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = c * 64 + tx * 4 + j;
        if (k < J) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float* p = A_s + k * kLLd + ty * 4 + i;
            *p = *p > 0.f ? dh[i][c * 4 + j] : 0.f;
          }
        }
      }
    __syncthreads();
    for (int i = tid; i < tT * J; i += kLThreads) {   // dE partial of frame t over the strip's columns, ascending u
      const int tt = i / J, k = i % J;
      const int t = t0 + tt;
      if (t >= T) continue;
      float s = 0.f;
      for (int uu = 0; uu < tU; ++uu) s += A_s[k * kLLd + tt * tU + uu];
      dE_part[((static_cast<int64_t>(strip) * B + b) * T + t) * J + k] = s;
    }
    for (int i = tid; i < tU * J; i += kLThreads) {   // dP of column u, ascending t
      const int uu = i / J, k = i % J;
      float s = dP_s[i];
      for (int tt = 0; tt < tT; ++tt) s += A_s[k * kLLd + tt * tU + uu];
      dP_s[i] = s;
    }
  }
  __syncthreads();
  for (int i = tid; i < tU * J; i += kLThreads) {
    const int u = u0 + i / J;
    if (u < U1) dP_part[((static_cast<int64_t>(range) * B + b) * U1 + u) * J + i % J] = dP_s[i];
  }
}

// ------------------------------------------------------------------ (3) class-major: dW_o / db_o partials
// grid (ceil(V1 / kLN), S).  Slice z: flattened node rows [z chunk, min(rows, (z + 1) chunk)), chunk a multiple of kLM.
// out: part [S][V1][J + 1] (column J: db) when S > 1, else dW [V1][J] / db [V1] directly.
template <int NC>
__global__ void __launch_bounds__(kLThreads) rnnt_loss_class_grad_kernel(
    const float* __restrict__ E, const float* __restrict__ P, const float* __restrict__ Wo, const float* __restrict__ bo,
    const int* __restrict__ targets, const int* __restrict__ enc_len, const int* __restrict__ target_len, const float* __restrict__ lse,
    const float* __restrict__ e_blank, const float* __restrict__ e_label, const float* __restrict__ grad, int T, int U, int J, int V1,
    int64_t rows, int64_t chunk, float* __restrict__ part, float* __restrict__ dW, float* __restrict__ db) {
  extern __shared__ float4 smem_f4[];
  constexpr int Arows = NC * 64;
  float* A_s = reinterpret_cast<float*>(smem_f4);   // [Arows][kLLd] relu(E + P), rows past J zero
  float* W_s = A_s + Arows * kLLd;                   // [kLK][kLLd]
  float* dz_s = W_s + kLK * kLLd;                    // [kLM][kLLd] dz, node-major
  __shared__ RowInfo ri;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int U1 = U + 1;
  const int n0 = blockIdx.x * kLN;
  const int64_t r_begin = static_cast<int64_t>(blockIdx.y) * chunk;
  const int64_t r_end = min(rows, r_begin + chunk);
  float dw[NC * 4][4];   // dw[c*4 + i][j]: joint unit c*64 + ty*4 + i, class n0 + tx*4 + j
  float dbv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < NC * 4; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) dw[c][j] = 0.f;
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kLM) {
    __syncthreads();   // the previous tile is done with A_s, dz_s and ri
    if (tid < kLM) {
      const int64_t r = r0 + tid;
      const int64_t bt = r / U1;
      stage_row(ri, tid, r < r_end, static_cast<int>(bt / T), static_cast<int>(bt % T), static_cast<int>(r % U1), T, U, enc_len,
                target_len, targets, lse, e_blank, e_label, grad);
    }
    __syncthreads();
    stage_hidden(A_s, Arows, ri, E, P, J, tid);
    float acc[4][4];
    logit_tile(A_s, W_s, Wo, n0, J, V1, tid, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dz_s[(ty * 4 + i) * kLLd + tx * 4 + j] = dz_of(ri, ty * 4 + i, n0 + tx * 4 + j, acc[i][j], bo, V1);
    __syncthreads();
#pragma unroll 4
    for (int m = 0; m < kLM; ++m) {   // ascending nodes
      const float4 a = *reinterpret_cast<const float4*>(dz_s + m * kLLd + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) dbv[j] += av[j];
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float h = A_s[(c * 64 + ty * 4 + i) * kLLd + m];
#pragma unroll
          for (int j = 0; j < 4; ++j) dw[c * 4 + i][j] = fmaf(h, av[j], dw[c * 4 + i][j]);
        }
    }
  }
  const int Kc = J + 1;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = n0 + tx * 4 + j;
    if (n >= V1) continue;
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int k = c * 64 + ty * 4 + i;
        if (k >= J) continue;
        if (part != nullptr)
          part[(static_cast<int64_t>(blockIdx.y) * V1 + n) * Kc + k] = dw[c * 4 + i][j];
        else
          dW[static_cast<int64_t>(n) * J + k] = dw[c * 4 + i][j];
      }
    if (ty == 0) {
      if (part != nullptr)
        part[(static_cast<int64_t>(blockIdx.y) * V1 + n) * Kc + J] = dbv[j];
      else
        db[n] = dbv[j];
    }
  }
}

constexpr size_t node_smem_bytes(int J, int tU) {
  return (static_cast<size_t>(loss_kpad(J)) * kLLd + kLK * kLLd + kLN * kLLd + kLK * loss_nc(J) * 64 + static_cast<size_t>(tU) * J) * 4;
}
constexpr size_t class_smem_bytes(int J) { return (static_cast<size_t>(loss_nc(J)) * 64 * kLLd + kLK * kLLd + kLM * kLLd) * 4; }
constexpr size_t kLossMaxSmem = 227 * 1024 - sizeof(RowInfo);

// the widest J (a multiple of 4) both gradient kernels hold in registers and shared memory at every strip width
constexpr int loss_max_hidden() {
  int J = 4;
  while (loss_nc(J + 4) <= kLMaxNC && node_smem_bytes(J + 4, kLM) <= kLossMaxSmem && class_smem_bytes(J + 4) <= kLossMaxSmem) J += 4;
  return J;
}
static_assert(loss_max_hidden() == GAM_RNNT_LOSS_MAX_JOINT_HIDDEN, "the header's joint_hidden limit of the fused loss");
static_assert(node_smem_bytes(GAM_RNNT_LOSS_MAX_JOINT_HIDDEN, kLM) == kLossMaxSmem,
              "at the widest joint the node kernel uses all of its shared memory (DESIGN.md section 4)");

template <int NC>
int launch_grads(const RnntLossArgs& a, const RnntLossPlan& p, float* dE_part, float* dP_part, float* part, float* dW, float* db,
                 cudaStream_t s) {
  static PerDeviceOnce attr_once;
  const size_t node_smem = node_smem_bytes(a.J, p.tU), class_smem = class_smem_bytes(a.J);
  if (attr_once.first() &&
      (cudaFuncSetAttribute(rnnt_loss_node_grad_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            static_cast<int>(kLossMaxSmem)) != cudaSuccess ||
       cudaFuncSetAttribute(rnnt_loss_class_grad_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            static_cast<int>(kLossMaxSmem)) != cudaSuccess))
    return -1;
  if (dE_part != nullptr) {
    const int n_tiles = (a.T + p.tT - 1) / p.tT;
    const int chunk = (n_tiles + p.ST - 1) / p.ST;
    rnnt_loss_node_grad_kernel<NC><<<dim3(p.NS, p.ST, a.B), kLThreads, node_smem, s>>>(
        a.E, a.P, a.Wo, a.bo, a.targets, a.enc_len, a.target_len, a.lse, a.e_blank, a.e_label, a.grad, a.B, a.T, a.U, a.J, a.V1, p.tU,
        chunk, dE_part, dP_part);
  }
  if (dW != nullptr) {
    const int64_t rows = static_cast<int64_t>(a.B) * a.T * (a.U + 1);
    int64_t chunk = (rows + p.S - 1) / p.S;
    chunk = (chunk + kLM - 1) / kLM * kLM;
    rnnt_loss_class_grad_kernel<NC><<<dim3((a.V1 + kLN - 1) / kLN, p.S), kLThreads, class_smem, s>>>(
        a.E, a.P, a.Wo, a.bo, a.targets, a.enc_len, a.target_len, a.lse, a.e_blank, a.e_label, a.grad, a.T, a.U, a.J, a.V1, rows, chunk,
        p.S > 1 ? part : nullptr, dW, db);
    if (p.S > 1) launch_outer_sum_reduce(part, p.S, a.V1, a.J, a.J + 1, dW, db, s);
  }
  return 0;
}

}  // namespace

int rnnt_loss_max_hidden() { return loss_max_hidden(); }

RnntLossPlan rnnt_loss_plan(int B, int T, int U, int V1) {
  RnntLossPlan p;
  const int U1 = U + 1;
  p.tU = 1;
  while (p.tU < U1 && p.tU < kLM) p.tU *= 2;
  p.tT = kLM / p.tU;
  p.NS = (U1 + p.tU - 1) / p.tU;
  const int n_tiles = (T + p.tT - 1) / p.tT;
  // about four waves of one-CTA-per-SM blocks on 132 SMs; every range keeps at least one frame tile
  int64_t st = (528 + static_cast<int64_t>(B) * p.NS - 1) / (static_cast<int64_t>(B) * p.NS);
  st = st < 1 ? 1 : (st > 64 ? 64 : st);
  p.ST = static_cast<int>(st < n_tiles ? st : n_tiles);
  const int64_t class_tiles = (V1 + kLN - 1) / kLN;
  const int64_t node_tiles = (static_cast<int64_t>(B) * T * U1 + kLM - 1) / kLM;
  int64_t S = (528 + class_tiles - 1) / class_tiles;
  S = S < 1 ? 1 : (S > 64 ? 64 : S);
  p.S = static_cast<int>(S < node_tiles ? S : node_tiles);
  return p;
}

int launch_rnnt_loss_alpha_beta(const float* blank, const float* label, const int* enc_len, const int* target_len, int B, int T, int U,
                                float* alpha, float* e_blank, float* e_label, float* loss, cudaStream_t s) {
  const int U1 = U + 1;
  const int threads = U1 <= 64 ? 64 : U1 >= 1024 ? 1024 : (U1 + 31) / 32 * 32;
  rnnt_loss_alpha_beta_kernel<<<B, threads, static_cast<size_t>(2) * U1 * 4, s>>>(blank, label, enc_len, target_len, T, U, alpha,
                                                                                  e_blank, e_label, loss);
  return 0;
}

int launch_rnnt_loss_grads(const RnntLossArgs& a, const RnntLossPlan& p, float* dE_part, float* dP_part, float* part, float* dW, float* db,
                           cudaStream_t s) {
  if (a.J % 4 != 0 || a.J > rnnt_loss_max_hidden()) return 1;
  switch (loss_nc(a.J)) {
    case 1: return launch_grads<1>(a, p, dE_part, dP_part, part, dW, db, s);
    case 2: return launch_grads<2>(a, p, dE_part, dP_part, part, dW, db, s);
    case 3: return launch_grads<3>(a, p, dE_part, dP_part, part, dW, db, s);
    case 4: return launch_grads<4>(a, p, dE_part, dP_part, part, dW, db, s);
    case 5: return launch_grads<5>(a, p, dE_part, dP_part, part, dW, db, s);
    case 6: return launch_grads<6>(a, p, dE_part, dP_part, part, dW, db, s);
    default: return 1;
  }
}

}  // namespace gam
