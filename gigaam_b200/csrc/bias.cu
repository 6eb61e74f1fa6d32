// Hotwords for CTC greedy output (include/gigaam_b200.h, gam_ctc_bias, has the definition): the detections of gam_ctc_spot
// that start and end on word boundaries replace the greedy tokens they cover, best gain first, without overlaps.
//   select  one CTA per recording.  Every stored detection's replaced range and eligibility are computed; the eligible ones are
//           compacted (block scans, so their order is fixed) into the workspace and bitonic-sorted on (gain, start, keyword
//           rank), a total order.  Thread 0 walks that order against a per-frame occupancy bitmap; the accepted spans are
//           listed in start order, identities are recognised, the replaced greedy tokens are struck from the per-frame table
//           and the path score is summed in start order in fp64.
//   trace   kBiasTraceCtas x 4 warps per recording stride over the accepted spans (no host read of their number).  A warp runs
//           the keyword's Viterbi over [s, e) from state 0 at s with ctc_spot_kernel's lane layout (4 states per lane) and
//           recursion, keeps 2-bit backpointers per (frame, state) at the recording's frame offset (32 bytes per frame: the
//           spans are disjoint), then lane 0 walks back from state S - 1 at e - 1, writes each keyword token at the first frame
//           of its run and adjusts frame_logp.
//   compact one CTA per recording: a block scan over frames merges the kept greedy tokens and the spliced ones into the
//           outputs.  Each frame holds a group of greedy tokens written before its spliced token and a group written after it:
//           the spaces kept at a splice's left edge form the group before frame s (select moves them there), those at its
//           right edge that do not follow the keyword's last token form the group after that token's frame (trace moves
//           them there), so a kept space never falls inside a spliced keyword.
// Fixed orders everywhere and no atomics: the outputs are a function of the recording's inputs alone.
#include <cmath>
#include <cstdint>

#include "kernels.h"

namespace gam {
namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kBiasThreads = 1024;
constexpr int kTraceWarps = 4;

// one recording's workspace, in 32-bit words from its base
struct BiasWs {
  int4* keys;            // [P] sort keys (~bits(G), s, keyword rank, candidate)
  int* kg;               // [T] first greedy token written at frame t before its spliced token, -1 when none
  int* kg_n;             // [T] how many (consecutive) greedy tokens from kg[t]
  int* ka;               // [T] first greedy token written at frame t after its spliced token, -1 when none
  int* ka_n;             // [T] how many from ka[t]
  int* kgsrc;            // [T] keyword of a confirmed (identity) greedy token at its own frame, else -1
  int* ins_id;           // [T] spliced token starting at frame t, else -1
  int* ins_k;            // [T] its keyword
  int* acc_at;           // [T] candidate of the accepted span starting at t, else -1
  int* acc_list;         // [T] accepted candidates in start order; identities as -1 - candidate
  float* mrow;           // [T] m[t] of traced frames
  uint32_t* occupied;    // [ceil(T / 32)] bitmap of accepted frames
  int* rank;             // [K] keyword order: longer first, then smaller ids, then index
  int* scalars;          // [4] eligible count, accepted count
  unsigned char* bp;     // [T, 32] backpointers, byte l of frame t = lane l's four states
};

__host__ __device__ inline int64_t next_pow2(int64_t n) {
  int64_t p = 1;
  while (p < n) p <<= 1;
  return p;
}

__host__ __device__ inline int64_t bias_candidates(int T, int K, int max_det) {
  return static_cast<int64_t>(K) * (max_det < T ? max_det : T);
}

__device__ inline BiasWs bias_ws(int32_t* base, int T, int K, int max_det) {
  BiasWs w;
  const int64_t P = next_pow2(bias_candidates(T, K, max_det));
  int32_t* p = base;
  w.keys = reinterpret_cast<int4*>(p);
  p += 4 * P;
  const int64_t T64 = T;
  w.kg = p;
  w.kg_n = p + T64;
  w.ka = p + 2 * T64;
  w.ka_n = p + 3 * T64;
  w.kgsrc = p + 4 * T64;
  w.ins_id = p + 5 * T64;
  w.ins_k = p + 6 * T64;
  w.acc_at = p + 7 * T64;
  w.acc_list = p + 8 * T64;
  w.mrow = reinterpret_cast<float*>(p + 9 * T64);
  p += 10 * T64;
  w.occupied = reinterpret_cast<uint32_t*>(p);
  p += (T + 31) / 32;
  w.rank = p;
  p += K;
  w.scalars = p;
  p += 4;
  w.bp = reinterpret_cast<unsigned char*>(p);
  return w;
}

// exclusive block scan of one int per thread (blockDim.x == kBiasThreads); *total receives the sum.  Ends synchronised.
__device__ int block_scan(int x, int* total) {
  __shared__ int warp_sum[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = x;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int y = __shfl_up_sync(kFull, inc, off);
    if (lane >= off) inc += y;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = warp_sum[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int y = __shfl_up_sync(kFull, w, off);
      if (lane >= off) w += y;
    }
    warp_sum[lane] = w;
  }
  __syncthreads();
  const int before = (warp ? warp_sum[warp - 1] : 0) + inc - x;
  *total = warp_sum[31];
  __syncthreads();
  return before;
}

__device__ inline bool key_less(const int4& a, const int4& b) {
  const unsigned ga = static_cast<unsigned>(a.x), gb = static_cast<unsigned>(b.x);
  if (ga != gb) return ga < gb;
  if (a.y != b.y) return a.y < b.y;
  return a.z < b.z;
}

// keyword a before keyword b in the last tie-breaks: the longer one, then the lexicographically smaller ids, then the index
__device__ bool keyword_before(const int* keywords, const int* keyword_len, int Umax, int a, int b) {
  const int ua = min(max(keyword_len[a], 0), Umax), ub = min(max(keyword_len[b], 0), Umax);
  if (ua != ub) return ua > ub;
  const int* ya = keywords + static_cast<int64_t>(a) * Umax;
  const int* yb = keywords + static_cast<int64_t>(b) * Umax;
  for (int i = 0; i < ua; ++i)
    if (ya[i] != yb[i]) return ya[i] < yb[i];
  return a < b;
}

__device__ inline int lower_bound(const int* f, int n, int x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (f[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ inline unsigned flag_of(const unsigned char* flags, int V, int id) { return id >= 0 && id < V ? flags[id] : 0u; }

// the replaced range [i0, i1) of span [s, e) with its edge spaces removed; false when it is empty or not on word boundaries
__device__ bool replaced_range(const int* ids, const int* fr, int n, const unsigned char* flags, int V, int s, int e, int* i0p, int* i1p) {
  int i0 = lower_bound(fr, n, s), i1 = lower_bound(fr, n, e);
  while (i0 < i1 && (flag_of(flags, V, ids[i0]) & 1u)) ++i0;
  while (i1 > i0 && (flag_of(flags, V, ids[i1 - 1]) & 1u)) --i1;
  if (i1 <= i0) return false;
  auto boundary = [&](int p) {
    return p == 0 || p == n || (flag_of(flags, V, ids[p - 1]) & 1u) || (flag_of(flags, V, ids[p]) & 3u);
  };
  *i0p = i0;
  *i1p = i1;
  return boundary(i0) && boundary(i1);
}

__global__ void __launch_bounds__(kBiasThreads) ctc_bias_select_kernel(BiasArgs a, int32_t* workspace, int64_t ws_words) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = a.T, K = a.K, max_det = a.max_det, V = a.V1 - 1;
  BiasWs w = bias_ws(workspace + b * ws_words, T, K, max_det);
  const int Tb = min(max(a.enc_len[b], 0), T);
  const int n = min(max(a.counts[b], 0), a.max_out);
  const int* ids = a.ids + static_cast<int64_t>(b) * a.max_out;
  const int* fr = a.frames + static_cast<int64_t>(b) * a.max_out;

  for (int t = tid; t < T; t += kBiasThreads) {
    w.kg[t] = w.ka[t] = w.kgsrc[t] = w.ins_id[t] = w.ins_k[t] = w.acc_at[t] = -1;
    w.kg_n[t] = 1;
    w.ka_n[t] = 0;
  }
  for (int i = tid; i < (T + 31) / 32; i += kBiasThreads) w.occupied[i] = 0u;
  for (int k = tid; k < K; k += kBiasThreads) {
    int r = 0;
    for (int j = 0; j < K; ++j) r += keyword_before(a.keywords, a.keyword_len, a.Umax, j, k);
    w.rank[k] = r;
  }
  __syncthreads();
  for (int i = tid; i < n; i += kBiasThreads)
    if (fr[i] >= 0 && fr[i] < T) w.kg[fr[i]] = i;

  // ---- eligible candidates, compacted in candidate order.  Spot's detections of one keyword are disjoint, so at most
  // min(max_det, T) of them are eligible and the key region holds them all; keys past it (detections that break that
  // contract) are dropped rather than written out of bounds.
  const int64_t N = static_cast<int64_t>(K) * max_det;
  const int cap = static_cast<int>(next_pow2(bias_candidates(T, K, max_det)));
  int n_elig = 0;
  for (int64_t base = 0; base < N; base += kBiasThreads) {
    const int64_t c = base + tid;
    int4 key = make_int4(0, 0, 0, 0);
    int ok = 0;
    if (c < N) {
      const int k = static_cast<int>(c / max_det), j = static_cast<int>(c % max_det);
      const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + j;
      const int U = a.keyword_len[k];
      if (j < min(a.det_count[static_cast<int64_t>(b) * K + k], max_det) && U >= 1 && U <= a.Umax) {
        const int s = a.det_start[row], e = a.det_end[row];
        const float G = a.det_score[row] - static_cast<float>(U) * a.log_theta;
        int i0, i1;
        if (G >= 0.f && s >= 0 && s < e && e <= Tb && replaced_range(ids, fr, n, a.flags, V, s, e, &i0, &i1)) {
          ok = 1;
          key = make_int4(static_cast<int>(~__float_as_uint(G + 0.f)), s, w.rank[k], static_cast<int>(c));
        }
      }
    }
    int total;
    const int pos = block_scan(ok, &total);
    if (ok && pos < cap - n_elig) w.keys[n_elig + pos] = key;
    n_elig = min(n_elig + total, cap);
  }
  // ---- bitonic sort of the padded power of two (sentinels sort last)
  const int P = static_cast<int>(next_pow2(n_elig));
  for (int i = n_elig + tid; i < P; i += kBiasThreads) w.keys[i] = make_int4(-1, 0x7fffffff, 0x7fffffff, -1);
  __syncthreads();
  for (int k2 = 2; k2 <= P; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += kBiasThreads) {
        const int l = i ^ j;
        if (l > i) {
          const int4 x = w.keys[i], y = w.keys[l];
          if ((i & k2) == 0 ? key_less(y, x) : key_less(x, y)) {
            w.keys[i] = y;
            w.keys[l] = x;
          }
        }
      }
      __syncthreads();
    }
  }
  // ---- the walk: accept a span that overlaps no accepted one
  if (tid == 0) {
    for (int i = 0; i < n_elig; ++i) {
      const int c = w.keys[i].w;
      const int64_t row = (static_cast<int64_t>(b) * K + c / max_det) * max_det + c % max_det;
      const int s = a.det_start[row], e = a.det_end[row];
      bool free_span = true;
      for (int t = s; t < e && free_span;) {
        const int bits = min(32 - (t & 31), e - t);
        const uint32_t mask = (bits == 32 ? kFull : ((1u << bits) - 1u)) << (t & 31);
        free_span = (w.occupied[t >> 5] & mask) == 0u;
        t += bits;
      }
      if (!free_span) continue;
      for (int t = s; t < e;) {
        const int bits = min(32 - (t & 31), e - t);
        w.occupied[t >> 5] |= (bits == 32 ? kFull : ((1u << bits) - 1u)) << (t & 31);
        t += bits;
      }
      w.acc_at[s] = c;
    }
  }
  __syncthreads();
  // ---- accepted spans in start order; identities keep the greedy tokens, the others strike them
  int n_acc = 0;
  for (int base = 0; base < T; base += kBiasThreads) {
    const int t = base + tid;
    const int c = t < T ? w.acc_at[t] : -1;
    int total;
    const int pos = block_scan(c >= 0, &total);
    if (c >= 0) {
      const int k = c / max_det;
      const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + c % max_det;
      int i0 = 0, i1 = 0;
      replaced_range(ids, fr, n, a.flags, V, a.det_start[row], a.det_end[row], &i0, &i1);
      const int U = a.keyword_len[k];
      const int* y = a.keywords + static_cast<int64_t>(k) * a.Umax;
      bool same = i1 - i0 == U;
      for (int i = 0; same && i < U; ++i) same = ids[i0 + i] == y[i];
      for (int i = i0; i < i1; ++i) {
        if (same) w.kgsrc[fr[i]] = k;
        else w.kg[fr[i]] = -1;
      }
      if (!same) {   // the spaces kept at the left edge are written before the keyword, at its first frame s
        const int s = a.det_start[row], r0 = lower_bound(fr, n, s);
        for (int i = r0; i < i0; ++i) w.kg[fr[i]] = -1;
        if (i0 > r0) {
          w.kg[s] = r0;
          w.kg_n[s] = i0 - r0;
        }
      }
      w.acc_list[n_acc + pos] = same ? -1 - c : c;
    }
    n_acc += total;
  }
  __syncthreads();
  if (tid == 0) {
    w.scalars[0] = n_elig;
    w.scalars[1] = n_acc;
    if (a.path_logp) {
      double sum = static_cast<double>(a.path_logp[b]);
      for (int i = 0; i < n_acc; ++i) {
        const int c = w.acc_list[i];
        if (c >= 0) sum += static_cast<double>(a.det_score[(static_cast<int64_t>(b) * K + c / max_det) * max_det + c % max_det]);
      }
      a.out_path_logp[b] = static_cast<float>(sum);
    }
  }
}

__global__ void __launch_bounds__(32 * kTraceWarps) ctc_bias_trace_kernel(BiasArgs a, int32_t* workspace, int64_t ws_words) {
  const int lane = threadIdx.x & 31, b = blockIdx.y;
  const int T = a.T, K = a.K, max_det = a.max_det, V1 = a.V1, blank = V1 - 1;
  BiasWs w = bias_ws(workspace + b * ws_words, T, K, max_det);
  const int n_acc = w.scalars[1];
  const float* lp = a.log_probs + static_cast<int64_t>(b) * T * V1;
  for (int idx = blockIdx.x * kTraceWarps + (threadIdx.x >> 5); idx < n_acc; idx += gridDim.x * kTraceWarps) {
    const int c = w.acc_list[idx];
    if (c < 0) continue;   // an identity: nothing to trace
    const int k = c / max_det;
    const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + c % max_det;
    const int s0 = a.det_start[row], e0 = a.det_end[row];
    const int U = a.keyword_len[k], S = 2 * U - 1;
    const int* y = a.keywords + static_cast<int64_t>(k) * a.Umax;
    int lab[4];
    bool skip[4], live[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int s = 4 * lane + j;
      live[j] = s < S;
      lab[j] = blank;
      skip[j] = false;
      if (live[j] && !(s & 1)) {
        lab[j] = y[s >> 1];
        skip[j] = s >= 2 && y[s >> 1] != y[(s >> 1) - 1];
      }
    }
    float v[4];
    for (int t = s0; t < e0; ++t) {
      const float* r = lp + static_cast<int64_t>(t) * V1;
      float mx = -INFINITY;
      int nan = 0;
      for (int cl = lane; cl < V1; cl += 32) {
        const float x = r[cl];
        mx = fmaxf(mx, x);
        nan |= isnan(x);
      }
#pragma unroll
      for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(kFull, mx, off));
      if (__any_sync(kFull, nan)) mx = __int_as_float(0x7fc00000);
      const float mt = mx + 0.f;
      if (lane == 0) w.mrow[t] = mt;
      if (t == s0) {   // the path starts on state 0 at s: spot's fresh start, best = 0
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = (lane == 0 && j == 0) ? (r[lab[0]] - mt) + 0.f : -INFINITY;
        continue;
      }
      float pv3 = __shfl_up_sync(kFull, v[3], 1), pv2 = __shfl_up_sync(kFull, v[2], 1);
      if (lane == 0) pv3 = pv2 = -INFINITY;
      float nv[4];
      unsigned code = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float best = v[j];
        unsigned from = 0;
        const float c1 = j >= 1 ? v[j - 1] : pv3;
        if (c1 > best) { best = c1; from = 1; }
        if (skip[j]) {
          const float c2 = j >= 2 ? v[j - 2] : (j == 1 ? pv3 : pv2);
          if (c2 > best) { best = c2; from = 2; }
        }
        nv[j] = live[j] ? (r[lab[j]] - mt) + best : -INFINITY;
        code |= from << (2 * j);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = nv[j];
      w.bp[static_cast<int64_t>(t) * 32 + lane] = static_cast<unsigned char>(code);
    }
    __syncwarp();
    if (lane == 0) {
      int st = S - 1, last = s0;
      for (int t = e0 - 1; t >= s0; --t) {
        const int label = (st & 1) ? blank : y[st >> 1];
        if (a.frame_logp)
          a.frame_logp[b * a.frame_pitch + t] += static_cast<double>(lp[static_cast<int64_t>(t) * V1 + label]) - static_cast<double>(w.mrow[t]);
        int prev = st;
        if (t > s0) prev = st - ((w.bp[static_cast<int64_t>(t) * 32 + (st >> 2)] >> (2 * (st & 3))) & 3);
        if (!(st & 1) && (t == s0 || prev != st)) {   // the first frame of this token's run
          w.ins_id[t] = y[st >> 1];
          w.ins_k[t] = k;
          if (st == S - 1) last = t;
        }
        st = max(prev, 0);
      }
      // the spaces kept at the right edge at or before the keyword's last token are written after it, at its frame
      const int n = min(max(a.counts[b], 0), a.max_out);
      const int* ids = a.ids + static_cast<int64_t>(b) * a.max_out;
      const int* fr = a.frames + static_cast<int64_t>(b) * a.max_out;
      int i0 = 0, i1 = 0;
      replaced_range(ids, fr, n, a.flags, V1 - 1, s0, e0, &i0, &i1);
      int j = i1;
      for (; j < n && fr[j] < e0 && fr[j] <= last; ++j) w.kg[fr[j]] = -1;
      if (j > i1) {
        w.ka[last] = i1;
        w.ka_n[last] = j - i1;
      }
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kBiasThreads) ctc_bias_compact_kernel(BiasArgs a, int32_t* workspace, int64_t ws_words) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = a.T, V1 = a.V1;
  BiasWs w = bias_ws(workspace + b * ws_words, T, a.K, a.max_det);
  const int64_t o = static_cast<int64_t>(b) * a.max_out;
  const float* lp = a.log_probs + static_cast<int64_t>(b) * T * V1;
  const int* fr = a.frames + o;
  int count = 0;
  // greedy tokens [g, g + gn) written at frame t, from position pos on
  auto put_greedy = [&](int g, int gn, int t, int pos) {
    for (int i = 0; i < gn && pos + i < a.max_out; ++i) {
      a.out_ids[o + pos + i] = a.ids[o + g + i];
      a.out_frames[o + pos + i] = t;
      a.out_source[o + pos + i] = w.kgsrc[fr[g + i]];
      if (a.out_token_logp) a.out_token_logp[o + pos + i] = a.token_logp[o + g + i];
    }
  };
  for (int base = 0; base < T; base += kBiasThreads) {
    const int t = base + tid;
    const int g = t < T ? w.kg[t] : -1, x = t < T ? w.ins_id[t] : -1, ga = t < T ? w.ka[t] : -1;
    const int gn = g >= 0 ? w.kg_n[t] : 0, an = ga >= 0 ? w.ka_n[t] : 0;
    int total;
    int pos = count + block_scan(gn + (x >= 0) + an, &total);
    put_greedy(g, gn, t, pos);
    pos += gn;
    if (x >= 0 && pos < a.max_out) {
      a.out_ids[o + pos] = x;
      a.out_frames[o + pos] = t;
      a.out_source[o + pos] = w.ins_k[t];
      if (a.out_token_logp) a.out_token_logp[o + pos] = lp[static_cast<int64_t>(t) * V1 + x];
    }
    pos += x >= 0;
    put_greedy(ga, an, t, pos);
    count += total;
  }
  if (tid == 0) a.out_counts[b] = min(count, a.max_out);
}

}  // namespace

int64_t ctc_bias_workspace_words(int T, int K, int max_det) {
  const int64_t P = next_pow2(bias_candidates(T, K, max_det));
  if (P > (int64_t(1) << 30)) return -1;
  const int64_t words = 4 * P + 10 * static_cast<int64_t>(T) + (T + 31) / 32 + K + 4 + 8 * static_cast<int64_t>(T);
  return (words + 3) / 4 * 4;
}

void launch_ctc_bias(const BiasArgs& a, int32_t* workspace, int stage, cudaStream_t s) {
  const int64_t ws_words = ctc_bias_workspace_words(a.T, a.K, a.max_det);
  if (stage == 0) ctc_bias_select_kernel<<<a.B, kBiasThreads, 0, s>>>(a, workspace, ws_words);
  if (stage == 1) ctc_bias_trace_kernel<<<dim3(kBiasTraceCtas, a.B), 32 * kTraceWarps, 0, s>>>(a, workspace, ws_words);
  if (stage == 2) ctc_bias_compact_kernel<<<a.B, kBiasThreads, 0, s>>>(a, workspace, ws_words);
}

}  // namespace gam
