// Front end of the path:
//   (1) fused log-mel:  frame -> Hann window -> real DFT (symmetric-folded, fp32) -> |X|^2 -> mel
//       filterbank -> clamp -> ln, one kernel, nothing but the waveform read and the [B,64,M] write
//       touches HBM.  Mirrors gigaam/preprocess.py:43-98 (torchaudio MelSpectrogram, power=2,
//       center / reflect padding on the batch buffer, HTK filterbank taken from the checkpoint).
//   (2) subsampling stage 1: Conv2d(1->C, 3x3, stride 2, pad 1) + time masks + ReLU, written
//       channels-last [B, T1, F1, C] fp16 so that stage 2 can fetch its im2col operand with strided
//       TMA boxes (gigaam/encoder.py:59-70,111-123).
#include "kernels.h"
#include "launch.cuh"

namespace gam {
namespace {

// ---------------------------------------------------------------------------------------------
// log-mel.  Real DFT of a length-N frame f (N even) folded on its symmetry:
//   Re X[k] = sum_{n=0}^{N/2} s[n] cos(2 pi k n / N),  s[0]=f[0], s[N/2]=f[N/2], s[n]=f[n]+f[N-n]
//   Im X[k] = -sum_{n=1}^{N/2-1} d[n] sin(2 pi k n / N),                      d[n]=f[n]-f[N-n]
// Block = 64 frames of one utterance.  Thread tile = 4 frames x 13 bins (bins strided by 16) so the
// power |X|^2 is thread-local.  K = N/2+1 is streamed in chunks of kKC rows of the cos/sin tables.
constexpr int kFr = 64;       // frames per block
constexpr int kBinsPad = 208; // 13 * 16 >= 201
constexpr int kKC = 32;       // table rows per smem chunk

struct LogmelSmem {
  // phase 1: folded frames s/d [kFr][K] ; tables chunk
  // phase 2: power [kFr][kBinsPad] (aliases s/d) ; out tile [64 mel][kFr+1]
};

// mel.clamp_(1e-9, 1e9) of gigaam/preprocess.py:50: NaN stays NaN (fmaxf alone would turn it into 1e-9, i.e. silence)
__device__ __forceinline__ float clamp_power(float v) { return v != v ? v : fminf(fmaxf(v, 1e-9f), 1e9f); }

__global__ void __launch_bounds__(256) logmel_kernel(const float* __restrict__ wav, int n_samples, int n_frames,
                                                     const float* __restrict__ window, const float* __restrict__ tcos,
                                                     const float* __restrict__ tsin, const float* __restrict__ fb,
                                                     float* __restrict__ mel, int n_fft, int hop, int center, int n_mels) {
  extern __shared__ float sm[];
  const int K = n_fft / 2 + 1;        // folded length (201 for n_fft = 400)
  const int nbins = K;                // rfft bins
  const int KP = K | 1;               // odd pitch -> conflict-free column walks
  float* s_fold = sm;                 // [kFr][KP]
  float* d_fold = sm + kFr * KP;      // [kFr][KP]
  float* tc = d_fold + kFr * KP;      // [kKC][kBinsPad]
  float* ts = tc + kKC * kBinsPad;    // [kKC][kBinsPad]

  const int b = blockIdx.y;
  const int f0 = blockIdx.x * kFr;
  const float* x = wav + static_cast<size_t>(b) * n_samples;
  const int half = n_fft / 2;

  // ---- fold windowed frames into s / d
  for (int i = threadIdx.x; i < kFr * K; i += blockDim.x) {
    const int fr = i / K, n = i % K;
    const int frame = f0 + fr;
    float sv = 0.f, dv = 0.f;
    if (frame < n_frames) {
      auto sample = [&](int j) -> float {
        int idx = frame * hop + j - (center ? half : 0);
        if (center) {
          if (idx < 0) idx = -idx;
          if (idx >= n_samples) idx = 2 * (n_samples - 1) - idx;
        }
        return (idx >= 0 && idx < n_samples) ? x[idx] * __ldg(window + j) : 0.f;
      };
      const float a = sample(n);
      if (n == 0 || n == half) {
        sv = a;
      } else {
        const float c = sample(n_fft - n);
        sv = a + c;
        dv = a - c;
      }
    }
    s_fold[fr * KP + n] = sv;
    d_fold[fr * KP + n] = dv;
  }

  const int tx = threadIdx.x & 15;   // bin lane: bins tx + 16*j
  const int ty = threadIdx.x >> 4;   // frame group: frames ty*4 .. ty*4+3
  float re[4][13], im[4][13];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 13; ++j) { re[i][j] = 0.f; im[i][j] = 0.f; }

  for (int k0 = 0; k0 < K; k0 += kKC) {
    __syncthreads();
    for (int i = threadIdx.x; i < kKC * kBinsPad; i += blockDim.x) {
      const int kk = i / kBinsPad, bin = i % kBinsPad;
      const int n = k0 + kk;
      float c = 0.f, s = 0.f;
      if (n < K && bin < nbins) {
        c = __ldg(tcos + static_cast<size_t>(n) * nbins + bin);
        s = __ldg(tsin + static_cast<size_t>(n) * nbins + bin);
      }
      tc[i] = c;
      ts[i] = s;
    }
    __syncthreads();
    const int kmax = min(kKC, K - k0);
    for (int kk = 0; kk < kmax; ++kk) {
      float sv[4], dv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sv[i] = s_fold[(ty * 4 + i) * KP + k0 + kk];
        dv[i] = d_fold[(ty * 4 + i) * KP + k0 + kk];
      }
#pragma unroll
      for (int j = 0; j < 13; ++j) {
        const float c = tc[kk * kBinsPad + tx + 16 * j];
        const float s = ts[kk * kBinsPad + tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          re[i][j] = fmaf(sv[i], c, re[i][j]);
          im[i][j] = fmaf(dv[i], s, im[i][j]);
        }
      }
    }
  }
  __syncthreads();
  // ---- power spectrum into smem (aliases the folded frames)
  float* pw = sm;  // [kFr][kBinsPad + 1]
  constexpr int PP = kBinsPad + 1;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 13; ++j) pw[(ty * 4 + i) * PP + tx + 16 * j] = re[i][j] * re[i][j] + im[i][j] * im[i][j];
  __syncthreads();
  // ---- mel projection + log; thread = (mel m, 16 frames)
  float* ot = sm + kFr * PP;  // [n_mels][kFr + 1]
  for (int m = threadIdx.x % 64; m < n_mels; m += 64) {
    const int fg = threadIdx.x / 64;  // 0..3 -> frames fg*16..
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int k = 0; k < nbins; ++k) {
      const float w = __ldg(fb + static_cast<size_t>(k) * n_mels + m);
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = fmaf(pw[(fg * 16 + i) * PP + k], w, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) ot[m * (kFr + 1) + fg * 16 + i] = logf(clamp_power(acc[i]));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_mels * kFr; i += blockDim.x) {
    const int m = i / kFr, fr = i % kFr;
    if (f0 + fr < n_frames) mel[(static_cast<size_t>(b) * n_mels + m) * n_frames + f0 + fr] = ot[m * (kFr + 1) + fr];
  }
}

// ---------------------------------------------------------------------------------------------
// Subsampling stage 1: y[b,t1,f1,c] = relu(mask_t1( bias[c] + sum_{kt,kf} w[c,kt,kf] * mask_t0(mel)[b, 2f1+kf-1, 2t1+kt-1] ))
// mel is [B, F, M] (feature-major as produced by the front end); the conv runs on its transpose
// [B,1,M,F] (gigaam/encoder.py:609-611).  block = (t1, b); 256 threads; thread = 3 channels x all f1.
__global__ void __launch_bounds__(256) subsample_conv1_kernel(const float* __restrict__ mel, const int* __restrict__ len0,
                                                              const int* __restrict__ len1, const int* __restrict__ run1,
                                                              const float* __restrict__ w, const float* __restrict__ bias,
                                                              __half* __restrict__ out, int M, int F, int T1, int F1, int C) {
  constexpr int kTT = 8;                      // output time steps per block (weights stay in registers across them)
  __shared__ float patch[2 * kTT + 1][72];    // mel rows 2 t1_0 - 1 .. 2 t1_0 + 2 kTT - 1, features -1..F  (F <= 70)
  const int t1_0 = blockIdx.x * kTT, b = blockIdx.y;
  if (run1 != nullptr && t1_0 >= __ldg(run1 + b)) return;   // no kept stage-2 frame reads these rows (pack_plan_kernel)
  const int L0 = len0[b], L1 = len1[b];
  for (int i = threadIdx.x; i < (2 * kTT + 1) * (F + 2); i += blockDim.x) {
    const int rr = i / (F + 2), ff = i % (F + 2) - 1;
    const int t0 = 2 * t1_0 + rr - 1;
    float v = 0.f;
    if (t0 >= 0 && t0 < M && t0 < L0 && ff >= 0 && ff < F) v = mel[(static_cast<size_t>(b) * F + ff) * M + t0];
    patch[rr][ff + 1] = v;
  }
  __syncthreads();
  // thread = 8 consecutive channels x half of the f1 range: one 16-byte store per (t1, f1, thread), 512 contiguous
  // bytes per warp instruction -- the kernel is bound by the 1.5 GB it writes, not by its 9 MACs per output
  const int groups = C / 8;
  const int cg = threadIdx.x % groups, fh = threadIdx.x / groups;
  const int nfh = blockDim.x / groups;
  const int c = cg * 8;
  float wk[8][9], bb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int k = 0; k < 9; ++k) wk[i][k] = __ldg(w + (c + i) * 9 + k);
    bb[i] = __ldg(bias + c + i);
  }
  for (int tt = 0; tt < kTT; ++tt) {
    const int t1 = t1_0 + tt;
    if (t1 >= T1) break;
    const bool live = t1 < L1;
    __half* ob = out + (static_cast<size_t>(b) * T1 + t1) * F1 * C;
    for (int f1 = fh; f1 < F1; f1 += nfh) {
      float x[9];
#pragma unroll
      for (int kt = 0; kt < 3; ++kt)
#pragma unroll
        for (int kf = 0; kf < 3; ++kf) x[kt * 3 + kf] = patch[2 * tt + kt][2 * f1 + kf];
      uint32_t pk[4];
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        float a0 = bb[i], a1 = bb[i + 1];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          a0 = fmaf(wk[i][k], x[k], a0);
          a1 = fmaf(wk[i + 1][k], x[k], a1);
        }
        __half2 hh = live ? __floats2half2_rn(fmaxf(a0, 0.f), fmaxf(a1, 0.f)) : __floats2half2_rn(0.f, 0.f);
        pk[i >> 1] = *reinterpret_cast<uint32_t*>(&hh);
      }
      *reinterpret_cast<uint4*>(ob + static_cast<size_t>(f1) * C + c) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  }
}

// mel [B, F, M] f32 -> [B, M, F] f16, frames t >= len0[b] zeroed (the _mask_time before the first conv1d,
// gigaam/encoder.py:118).  32 x 32 smem transpose tiles.
__global__ void __launch_bounds__(256) mel_to_tmajor_f16_kernel(const float* __restrict__ mel, const int* __restrict__ len0,
                                                                __half* __restrict__ out, int F, int M) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 8 rows per pass
  const int L = len0[b];
  for (int i = ty; i < 32; i += 8) {
    const int f = f0 + i, t = t0 + tx;
    tile[i][tx] = (f < F && t < M && t < L) ? mel[(static_cast<size_t>(b) * F + f) * M + t] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, f = f0 + tx;
    if (t < M && f < F) out[(static_cast<size_t>(b) * M + t) * F + f] = __float2half_rn(tile[tx][i]);
  }
}

// ---------------------------------------------------------------------------------------------------------
// Tensor-core front end.  The real DFT of every windowed frame is a GEMM  X = F . D^T  (F: frames x n_fft,
// D: cos|sin basis); fp16 alone would bury quiet bins under rounding noise, so both operands are split into
// fp16 (hi, lo) pairs and the three significant products are folded into ONE GEMM by concatenating along K:
//   A' = [ f_hi | f_lo | f_hi ],   W' = [ d_hi | d_hi | d_lo ]     (K = 3 * Kp, ~22-bit effective mantissas)
// run on the wgmma GEMM kernel with the power epilogue (re^2 + im^2).  This kernel builds A'.
// Frame f is stored as x.w.2^e_f: e_f = 11 moves the fp16 `lo` halves of quiet samples out of the subnormal range, and
// is lowered for a frame whose max |x.w| (NaN ignored) would round a `hi` to inf, so that max |x.w.2^e_f| < 2^15.
// e_f goes to fexp[f]; the GEMM epilogue undoes 2^22 and mel_log_kernel the remaining 2^(2 e_f - 22).
constexpr int kSplitIters = 8;   // Kp / 64: gam_logmel_tc admits n_fft / 2 + 1 <= 256 bins, so Kp <= 512
__global__ void __launch_bounds__(256) frames_split_kernel(const float* __restrict__ wav, int n_samples, int n_frames,
                                                           const float* __restrict__ window, __half* __restrict__ A,
                                                           int* __restrict__ fexp, int n_fft, int Kp, int hop, int center) {
  const int b = blockIdx.y;
  const int frame = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (frame >= n_frames) return;
  const int lane = threadIdx.x & 31;
  const float* x = wav + static_cast<size_t>(b) * n_samples;
  const size_t f = static_cast<size_t>(b) * n_frames + frame;
  __half* row = A + f * (3 * Kp);
  const int half = n_fft / 2;
  float v[kSplitIters][2];
  float amax = 0.f;
#pragma unroll
  for (int it = 0; it < kSplitIters; ++it) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = 2 * (lane + 32 * it) + e;
      float s = 0.f;
      if (j < n_fft) {
        int idx = frame * hop + j - (center ? half : 0);
        if (center) {
          if (idx < 0) idx = -idx;
          if (idx >= n_samples) idx = 2 * (n_samples - 1) - idx;
        }
        if (idx >= 0 && idx < n_samples) s = x[idx] * __ldg(window + j);
      }
      v[it][e] = s;
      amax = fmaxf(amax, fabsf(s));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  // fp16 rounds [65520, inf) to inf; 2^11 is kept whenever it fits, so frames with |x| <= 1 are stored as before
  const int ef = amax * 2048.0f < 65520.0f ? 11 : max(14 - ilogbf(amax), -126);
  const float scale = __int_as_float((127 + ef) << 23);
  if (lane == 0) fexp[f] = ef;
#pragma unroll
  for (int it = 0; it < kSplitIters; ++it) {
    const int i2 = lane + 32 * it;
    if (i2 >= Kp / 2) break;
    const float v0 = v[it][0] * scale, v1 = v[it][1] * scale;
    const __half2 hi = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    reinterpret_cast<__half2*>(row)[i2] = hi;
    reinterpret_cast<__half2*>(row + Kp)[i2] = lo;
    reinterpret_cast<__half2*>(row + 2 * Kp)[i2] = hi;
  }
}

// power spectrum [F, ldp] f32 -> log(clamp(P . fb)) written as [B, n_mels, M] (gigaam/preprocess.py:49-50, MelScale).
// block = 32 frames of one utterance; thread = (mel m, 8 frames); the HTK triangles are sparse, so each mel filter only
// walks its own bin range [lo_m, hi_m).  Frame f's power rows carry 2^(2 fexp[f] - 22) (frames_split_kernel), undone exactly
// before the clamp.
__global__ void __launch_bounds__(256) mel_log_kernel(const float* __restrict__ P, const int* __restrict__ fexp, int ldp, int n_frames,
                                                      int nbins, const float* __restrict__ fb, const int* __restrict__ mel_lo,
                                                      const int* __restrict__ mel_hi, float* __restrict__ mel, int n_mels) {
  __shared__ float ps[32][257];
  __shared__ float ot[64][33];
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * 32;
  for (int i = threadIdx.x; i < 32 * 64; i += 256) {
    const int fr = i / 64, c4 = (i % 64) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (f0 + fr < n_frames && c4 < ldp) v = *reinterpret_cast<const float4*>(P + (static_cast<size_t>(b) * n_frames + f0 + fr) * ldp + c4);
    ps[fr][c4] = v.x; ps[fr][c4 + 1] = v.y; ps[fr][c4 + 2] = v.z; ps[fr][c4 + 3] = v.w;
  }
  __syncthreads();
  const int m = threadIdx.x & 63, fg = threadIdx.x >> 6;
  if (m < n_mels) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    const int lo = mel_lo[m], hi = min(mel_hi[m], nbins);
    for (int k = lo; k < hi; ++k) {
      const float w = __ldg(fb + static_cast<size_t>(k) * n_mels + m);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(ps[fg * 8 + i][k], w, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int fr = min(f0 + fg * 8 + i, n_frames - 1);   // rows past the last frame are zero and never stored
      ot[m][fg * 8 + i] = logf(clamp_power(ldexpf(acc[i], 22 - 2 * __ldg(fexp + static_cast<size_t>(b) * n_frames + fr))));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_mels * 32; i += 256) {
    const int mm = i / 32, fr = i % 32;
    if (f0 + fr < n_frames) mel[(static_cast<size_t>(b) * n_mels + mm) * n_frames + f0 + fr] = ot[mm][fr];
  }
}

}  // namespace

int launch_frames_split(const float* wav, int B, int n_samples, int n_frames, const float* window, __half* A, int* fexp, int n_fft,
                        int Kp, int hop, int center, cudaStream_t s) {
  if (Kp > 64 * kSplitIters || n_fft > Kp) return -1;
  dim3 grid((n_frames + 7) / 8, B);
  frames_split_kernel<<<grid, 256, 0, s>>>(wav, n_samples, n_frames, window, A, fexp, n_fft, Kp, hop, center);
  return 0;
}

int launch_mel_log(const float* P, const int* fexp, int ldp, int B, int n_frames, int nbins, const float* fb, const int* mel_lo,
                   const int* mel_hi, float* mel, int n_mels, cudaStream_t s) {
  if (n_mels > 64 || nbins > 256 || ldp != 256) return -1;   // ot[64][33], ps[32][257] and its float4 row loads
  dim3 grid((n_frames + 31) / 32, B);
  mel_log_kernel<<<grid, 256, 0, s>>>(P, fexp, ldp, n_frames, nbins, fb, mel_lo, mel_hi, mel, n_mels);
  return 0;
}

void launch_mel_to_tmajor_f16(const float* mel, const int* len0, __half* out, int B, int F, int M, cudaStream_t s) {
  dim3 grid((M + 31) / 32, (F + 31) / 32, B);
  mel_to_tmajor_f16_kernel<<<grid, 256, 0, s>>>(mel, len0, out, F, M);
}

int logmel_smem_bytes(int n_fft) {
  const int K = n_fft / 2 + 1, KP = K | 1;
  const int phase1 = (2 * kFr * KP + 2 * kKC * kBinsPad) * 4;
  const int phase2 = (kFr * (kBinsPad + 1) + 64 * (kFr + 1)) * 4;
  return phase1 > phase2 ? phase1 : phase2;
}

int launch_logmel(const float* wav, int B, int n_samples, int n_frames, const float* window, const float* tcos,
                  const float* tsin, const float* fb, float* mel, int n_fft, int hop, int center, int n_mels,
                  cudaStream_t s) {
  if (n_fft / 2 + 1 > kBinsPad || n_mels > 64 || (n_fft & 1)) return -1;
  const int smem = logmel_smem_bytes(n_fft);
  static PerDeviceOnce attr_once;
  if (attr_once.first()) cudaFuncSetAttribute(logmel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  dim3 grid((n_frames + kFr - 1) / kFr, B);
  logmel_kernel<<<grid, 256, smem, s>>>(wav, n_samples, n_frames, window, tcos, tsin, fb, mel, n_fft, hop, center, n_mels);
  return 0;
}

int launch_subsample_conv1(const float* mel, const int* len0, const int* len1, const int* run1, const float* w, const float* bias,
                           __half* out, int B, int M, int F, int T1, int F1, int C, cudaStream_t s) {
  if (F > 70 || C % 8 != 0 || C / 8 > 128) return -1;
  dim3 grid((T1 + 7) / 8, B);
  subsample_conv1_kernel<<<grid, 2 * (C / 8), 0, s>>>(mel, len0, len1, run1, w, bias, out, M, F, T1, F1, C);
  return 0;
}

}  // namespace gam
