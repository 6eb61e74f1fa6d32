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
// Resumable (gam_ctc_bias_resume): the rows, greedy tokens and detections cover stream frames [frame_base, frame_base + hi), held
// by the caller.  Select first finds the horizon h (the earliest start of a spot path that can still become a detection, from
// the spot records), the first undecided overlap component D (one whose last end is past h or past the last greedy token)
// and the release frame R = min(h, D); only candidates starting before D take part, compact writes frames < R, and the
// candidates from D on are carried out.  A one-shot call (gam_ctc_bias) is a finished resume from frame 0.
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
  int* scalars;          // [4] eligible count, accepted count, release frame R, first undecided start D
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

// the block's minimum of one int per thread (blockDim.x == kBiasThreads).  Ends synchronised.
__device__ int block_min(int x) {
  __shared__ int warp_min[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  x = __reduce_min_sync(kFull, x);
  if (lane == 0) warp_min[warp] = x;
  __syncthreads();
  x = __reduce_min_sync(kFull, warp_min[lane]);
  __syncthreads();
  return x;
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

// the replaced range [i0, i1) of span [s, e) with its edge spaces removed; false when it is empty or not on word boundaries.
// left / right: whether the first / past-the-last token position is a word boundary (the start and end of a whole recording
// are; a held range starts on one when the stream does or the last greedy token before it is a space, and ends on one only
// when the stream finishes)
__device__ bool replaced_range(const int* ids, const int* fr, int n, const unsigned char* flags, int V, int s, int e, bool left,
                               bool right, int* i0p, int* i1p) {
  int i0 = lower_bound(fr, n, s), i1 = lower_bound(fr, n, e);
  while (i0 < i1 && (flag_of(flags, V, ids[i0]) & 1u)) ++i0;
  while (i1 > i0 && (flag_of(flags, V, ids[i1 - 1]) & 1u)) --i1;
  if (i1 <= i0) return false;
  auto boundary = [&](int p) {
    return (p == 0 ? left : (flag_of(flags, V, ids[p - 1]) & 1u) != 0) || (p == n ? right : (flag_of(flags, V, ids[p]) & 3u) != 0);
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
  // stream frame base + t is local frame t; a one-shot call is a finished stream from frame 0
  const bool resume = a.frame_base != nullptr;
  const int base = resume ? a.frame_base[b] : 0;
  const bool fin = !resume || a.finish[b] != 0, left = !resume || a.left_boundary[b] != 0;

  for (int t = tid; t < T; t += kBiasThreads) {
    w.kg[t] = w.ka[t] = w.kgsrc[t] = w.ins_id[t] = w.ins_k[t] = w.acc_at[t] = w.acc_list[t] = -1;
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
    if (fr[i] - base >= 0 && fr[i] - base < T) w.kg[fr[i] - base] = i;

  // ---- what is decided (local frames).  Finished: everything, R = T_b.  Otherwise the horizon h: spot costs are <= 0, so a
  // path that will end as a candidate (E >= tau) has v >= tau now, and every detection not yet emitted starts at or after
  // the start of the pending one or of a state with v >= tau (NaN fails), or at a later frame.  A component of the known
  // candidates' overlap graph is decided when it ends at or before h and at or before the last greedy token's frame (its
  // members' right boundaries are known); the decided ones form a prefix in time, and D is the start of the first other one.
  int D = Tb, R = Tb;
  if (!fin) {
    const int L4 = (2 * a.Umax - 1 + 3) / 4, per = 2 * a.Umax - 1;
    int hmin = Tb;
    for (int64_t i = tid; i < static_cast<int64_t>(K) * per; i += kBiasThreads) {
      const int k = static_cast<int>(i / per), st = static_cast<int>(i % per), U = a.keyword_len[k];
      if (U < 1 || U > a.Umax || st >= 2 * U - 1) continue;
      const SpotRecord* rec = reinterpret_cast<const SpotRecord*>(a.state + (static_cast<int64_t>(b) * K + k) * a.record);
      const float* v = reinterpret_cast<const float*>(rec + 1);
      const int* from = reinterpret_cast<const int*>(v + 4 * L4);
      const int at = (st & 3) * L4 + (st >> 2);
      if (v[at] >= static_cast<float>(U) * a.log_theta) hmin = min(hmin, from[at] - base);
      if (st == 0 && rec->has) hmin = min(hmin, rec->p_start - base);
    }
    const int h = max(block_min(hmin), 0);
    if (tid == 0) {
      // acc_list[t] holds, until the walk, the latest end of the known candidates starting at local frame t
      for (int k = 0; k < K; ++k)
        for (int j = 0; j < min(a.det_count[static_cast<int64_t>(b) * K + k], max_det); ++j) {
          const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + j;
          const int s = a.det_start[row] - base, e = a.det_end[row] - base;
          if (s >= 0 && s < e && e <= Tb) w.acc_list[s] = max(w.acc_list[s], e);
        }
      const int last = min(h, n > 0 ? fr[n - 1] - base : -1);
      int c0 = 0, c1 = -1;   // the current component [c0, c1)
      for (int t = 0; t < Tb && D == Tb; ++t) {
        const int e = w.acc_list[t];
        if (e < 0) continue;
        if (t >= c1) {
          if (c1 > last) D = c0;
          c0 = t;
          c1 = e;
        } else {
          c1 = max(c1, e);
        }
      }
      if (D == Tb && c1 > last) D = c0;
      w.scalars[2] = min(h, D);
      w.scalars[3] = D;
    }
    __syncthreads();
    R = w.scalars[2];
    D = w.scalars[3];
    for (int t = tid; t < T; t += kBiasThreads) w.acc_list[t] = -1;
    __syncthreads();
  } else if (tid == 0) {
    w.scalars[2] = R;
  }

  // ---- eligible candidates, compacted in candidate order.  Spot's detections of one keyword are disjoint, so at most
  // min(max_det, T) of them are eligible and the key region holds them all; keys past it (detections that break that
  // contract) are dropped rather than written out of bounds.
  const int64_t N = static_cast<int64_t>(K) * max_det;
  const int cap = static_cast<int>(next_pow2(bias_candidates(T, K, max_det)));
  int n_elig = 0;
  for (int64_t c0 = 0; c0 < N; c0 += kBiasThreads) {
    const int64_t c = c0 + tid;
    int4 key = make_int4(0, 0, 0, 0);
    int ok = 0;
    if (c < N) {
      const int k = static_cast<int>(c / max_det), j = static_cast<int>(c % max_det);
      const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + j;
      const int U = a.keyword_len[k];
      if (j < min(a.det_count[static_cast<int64_t>(b) * K + k], max_det) && U >= 1 && U <= a.Umax) {
        const int s = a.det_start[row] - base, e = a.det_end[row] - base;
        const float G = a.det_score[row] - static_cast<float>(U) * a.log_theta;
        int i0, i1;
        if (G >= 0.f && s >= 0 && s < e && e <= Tb && s < D &&
            replaced_range(ids, fr, n, a.flags, V, s + base, e + base, left, fin, &i0, &i1)) {
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
      const int s = a.det_start[row] - base, e = a.det_end[row] - base;
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
  for (int t0 = 0; t0 < T; t0 += kBiasThreads) {
    const int t = t0 + tid;
    const int c = t < T ? w.acc_at[t] : -1;
    int total;
    const int pos = block_scan(c >= 0, &total);
    if (c >= 0) {
      const int k = c / max_det;
      const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + c % max_det;
      int i0 = 0, i1 = 0;
      replaced_range(ids, fr, n, a.flags, V, a.det_start[row], a.det_end[row], left, fin, &i0, &i1);
      const int U = a.keyword_len[k];
      const int* y = a.keywords + static_cast<int64_t>(k) * a.Umax;
      bool same = i1 - i0 == U;
      for (int i = 0; same && i < U; ++i) same = ids[i0 + i] == y[i];
      for (int i = i0; i < i1; ++i) {
        const int f = fr[i] - base;
        if (f < 0 || f >= T) continue;   // a token outside the rows breaks the input contract: never written out of bounds
        if (same) w.kgsrc[f] = k;
        else w.kg[f] = -1;
      }
      if (!same) {   // the spaces kept at the left edge are written before the keyword, at its first frame s
        const int s = a.det_start[row] - base, r0 = lower_bound(fr, n, s + base);
        for (int i = r0; i < i0; ++i)
          if (fr[i] - base >= 0 && fr[i] - base < T) w.kg[fr[i] - base] = -1;
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
    if (resume) a.released_until[b] = base + R;
  }
  // ---- resume: the undecided candidates (those from D on), compacted in their order, for the next call
  if (resume) {
    for (int k = tid; k < K; k += kBiasThreads) {
      const int64_t row0 = (static_cast<int64_t>(b) * K + k) * max_det;
      int c = 0;
      for (int j = 0; j < min(a.det_count[static_cast<int64_t>(b) * K + k], max_det); ++j) {
        const int s = a.det_start[row0 + j] - base, e = a.det_end[row0 + j] - base;
        if (s >= D && s < e && e <= Tb) {
          a.carry_start[row0 + c] = a.det_start[row0 + j];
          a.carry_end[row0 + c] = a.det_end[row0 + j];
          a.carry_score[row0 + c] = a.det_score[row0 + j];
          ++c;
        }
      }
      a.carry_count[static_cast<int64_t>(b) * K + k] = c;
    }
  }
}

__global__ void __launch_bounds__(32 * kTraceWarps) ctc_bias_trace_kernel(BiasArgs a, int32_t* workspace, int64_t ws_words) {
  const int lane = threadIdx.x & 31, b = blockIdx.y;
  const int T = a.T, K = a.K, max_det = a.max_det, V1 = a.V1, blank = V1 - 1;
  BiasWs w = bias_ws(workspace + b * ws_words, T, K, max_det);
  const int n_acc = w.scalars[1];
  const int base = a.frame_base ? a.frame_base[b] : 0;
  const float* lp = a.log_probs + static_cast<int64_t>(b) * T * V1;
  for (int idx = blockIdx.x * kTraceWarps + (threadIdx.x >> 5); idx < n_acc; idx += gridDim.x * kTraceWarps) {
    const int c = w.acc_list[idx];
    if (c < 0) continue;   // an identity: nothing to trace
    const int k = c / max_det;
    const int64_t row = (static_cast<int64_t>(b) * K + k) * max_det + c % max_det;
    const int s0 = a.det_start[row] - base, e0 = a.det_end[row] - base;
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
      replaced_range(ids, fr, n, a.flags, V1 - 1, s0 + base, e0 + base, true, true, &i0, &i1);
      int j = i1;
      for (; j < n && fr[j] - base < e0 && fr[j] - base <= last; ++j)
        if (fr[j] - base >= 0) w.kg[fr[j] - base] = -1;
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
  const int base = a.frame_base ? a.frame_base[b] : 0;
  const int T_out = a.frame_base ? w.scalars[2] : T;   // a resume call writes the frames before its release frame
  int count = 0;
  // greedy tokens [g, g + gn) written at frame t, from position pos on
  auto put_greedy = [&](int g, int gn, int t, int pos) {
    for (int i = 0; i < gn && pos + i < a.max_out; ++i) {
      a.out_ids[o + pos + i] = a.ids[o + g + i];
      a.out_frames[o + pos + i] = base + t;
      const int f = fr[g + i] - base;
      a.out_source[o + pos + i] = f >= 0 && f < T ? w.kgsrc[f] : -1;
      if (a.out_token_logp) a.out_token_logp[o + pos + i] = a.token_logp[o + g + i];
    }
  };
  for (int t0 = 0; t0 < T_out; t0 += kBiasThreads) {
    const int t = t0 + tid;
    const int g = t < T_out ? w.kg[t] : -1, x = t < T_out ? w.ins_id[t] : -1, ga = t < T_out ? w.ka[t] : -1;
    const int gn = g >= 0 ? w.kg_n[t] : 0, an = ga >= 0 ? w.ka_n[t] : 0;
    int total;
    int pos = count + block_scan(gn + (x >= 0) + an, &total);
    put_greedy(g, gn, t, pos);
    pos += gn;
    if (x >= 0 && pos < a.max_out) {
      a.out_ids[o + pos] = x;
      a.out_frames[o + pos] = base + t;
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
