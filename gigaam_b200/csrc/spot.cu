// CTC keyword spotting over caller fp32 log-probs (include/gigaam_b200.h, gam_ctc_spot, has the definition).
// Grid (keyword groups, recordings); one warp per keyword, its S = 2U - 1 <= 127 states 4 to a lane (lane l owns states
// 4l .. 4l + 3), so the s - 1 / s - 2 predecessors of a lane's first two states come from lane l - 1 by shuffles.
// The recording's rows arrive in tiles of R contiguous frames, bulk-copied (cp.async.bulk) into a ring of kSpotStages
// shared-memory stages behind one mbarrier each, and every tile is shared by all keyword warps of the CTA.  Once a tile has
// landed, the warps compute each of its frames' m[t] = max_c lp[t, c] (NaN when the row holds a NaN) once for the CTA, one
// __syncthreads publishes them, and each warp then walks the tile's frames; the same barrier tells thread 0 that the stage
// read in the tile before is free, so it refills that stage kSpotStages tiles ahead.  The detection scan runs inside the walk
// (lane 0 stores a detection when it is emitted), so nothing of size T x K is stored.  A warp reads only its own keyword
// and the per-frame m, whose max is exact in any order: a (recording, keyword) pair gets the same bits in any batch, keyword
// order or warps-per-CTA choice.  No atomics, no host synchronisation.
// Resumable (gam_ctc_spot_resume): a row walks its local frames [lo, hi) as stream frames frame_base + t, and each warp loads
// its (stream, keyword) SpotRecord before the walk and stores it after, so a stream split into consecutive calls gives the
// one-shot bits.  A one-shot call (gam_ctc_spot) is the same walk from fresh registers over [0, enc_len) with finish.
#include <algorithm>
#include <cmath>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"
#include "rowmax.cuh"

namespace gam {
namespace {

constexpr int kSpotStages = 4;
constexpr int kSpotTileBytes = 16384;   // target bytes of log-probs per tile
constexpr int kSpotMaxRows = 32;        // frames per tile at most
constexpr int kSpotHeader = 1024;       // mbarriers at 0, m[t] of every stage at 128, tiles from here
constexpr unsigned kFull = 0xffffffffu;

// lanes of a record: those that own at least one of the 2 Umax - 1 states
__host__ __device__ constexpr int spot_record_lanes(int Umax) { return (2 * Umax - 1 + 3) / 4; }

__global__ void __launch_bounds__(1024) ctc_spot_kernel(const float* __restrict__ log_probs, const SpotResume io,
                                                        const int* __restrict__ keywords, const int* __restrict__ keyword_len, int T,
                                                        int V1, int K, int Umax, float log_theta, int max_det, int R, int stage_bytes,
                                                        int* __restrict__ det_start, int* __restrict__ det_end,
                                                        float* __restrict__ det_score, int* __restrict__ det_count) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  float* mrow = reinterpret_cast<float*>(smem + 128);   // [kSpotStages][R]
  unsigned char* tiles = smem + kSpotHeader;            // [kSpotStages][stage_bytes]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int b = blockIdx.y, k = blockIdx.x * nw + warp;
  // local frames [f0, Tb) of row b; frame t of the row is frame fb + t of its stream (0 on a fresh call)
  const bool resume = io.state != nullptr;
  const int Tb = min(max(io.hi[b], 0), T);
  const int f0 = resume ? min(max(io.lo[b], 0), Tb) : 0, fb = resume ? io.frame_base[b] : 0;
  const int blank = V1 - 1;

  // ---- this warp's keyword: labels of its lane's four states, and which even states may skip the blank before them
  int U = 0, bad = 1;
  const int* y = keywords + static_cast<int64_t>(min(k, K - 1)) * Umax;
  if (k < K) {
    U = keyword_len[k];
    bad = U < 1 || U > Umax;
    if (!bad) {
      int out = 0;
      for (int i = lane; i < U; i += 32) out |= y[i] < 0 || y[i] >= blank;
      bad = __any_sync(kFull, out);
    }
  }
  const bool active = k < K && !bad;
  const int S = 2 * U - 1;
  int lab[4];
  bool skip[4], live[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int s = 4 * lane + j;
    live[j] = active && s < S;
    lab[j] = blank;
    skip[j] = false;
    if (live[j] && !(s & 1)) {
      lab[j] = y[s >> 1];
      skip[j] = s >= 2 && y[s >> 1] != y[(s >> 1) - 1];
    }
  }
  const int e_lane = active ? (S - 1) >> 2 : 0, e_slot = active ? (S - 1) & 3 : 0;
  const float tau = static_cast<float>(U) * log_theta;
  const int64_t row0 = (static_cast<int64_t>(b) * K + min(k, K - 1)) * max_det;

  float v[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  int a[4] = {0, 0, 0, 0};
  int has = 0, p_start = 0, p_end = 0, total = 0;
  float p_score = 0.f;
  // the stream's record: loaded once before the frame walk, stored once after it
  const int L = spot_record_lanes(Umax);
  SpotRecord* rec = resume && k < K ? reinterpret_cast<SpotRecord*>(io.state + (static_cast<int64_t>(b) * K + k) * io.record) : nullptr;
  float* rec_v = rec ? reinterpret_cast<float*>(rec + 1) : nullptr;   // [4][L]
  int* rec_a = rec ? reinterpret_cast<int*>(rec_v + 4 * L) : nullptr;  // [4][L]
  if (rec && active) {
    has = rec->has;
    p_start = rec->p_start;
    p_end = rec->p_end;
    p_score = rec->p_score;
    total = rec->total;
    if (lane < L) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] = rec_v[j * L + lane];
        a[j] = rec_a[j * L + lane];
      }
    }
  }
  // detections stored so far: appended after the caller's count on a resume call
  const int base = resume && k < K ? min(max(det_count[static_cast<int64_t>(b) * K + k], 0), max_det) : 0;
  int count = base;
  auto emit = [&]() {
    if (lane == 0 && count < max_det) {
      det_start[row0 + count] = p_start;
      det_end[row0 + count] = p_end;
      det_score[row0 + count] = p_score;
    }
    ++count;
  };

  // ---- the tile ring
  if (tid == 0) {
    for (int i = 0; i < kSpotStages; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  const int any = __syncthreads_or(active);
  const int ntiles = any ? (Tb - f0 + R - 1) / R : 0;
  const float* lp = log_probs + (static_cast<int64_t>(b) * T + f0) * V1;
  // tile i: frames [i R, i R + n) copied from the 16-byte boundary at or below its first row up to the one at or above its
  // end; its first row lands `skew` bytes into the stage
  auto tile_src = [&](int i) { return reinterpret_cast<uintptr_t>(lp + static_cast<int64_t>(i) * R * V1); };
  auto issue = [&](int i) {
    const int st = i % kSpotStages, n = min(R, Tb - f0 - i * R);
    const uintptr_t lo = tile_src(i) & ~uintptr_t(15);
    const uintptr_t hi = (tile_src(i) + static_cast<uintptr_t>(n) * V1 * 4 + 15) & ~uintptr_t(15);
    ptx::mbar_arrive_expect_tx(&full[st], static_cast<uint32_t>(hi - lo));
    ptx::bulk_load(tiles + st * stage_bytes, reinterpret_cast<const void*>(lo), static_cast<uint32_t>(hi - lo), &full[st]);
  };
  if (tid == 0)
    for (int i = 0; i < min(kSpotStages, ntiles); ++i) issue(i);

  for (int i = 0; i < ntiles; ++i) {
    const int st = i % kSpotStages, n = min(R, Tb - f0 - i * R);
    ptx::mbar_wait(&full[st], (i / kSpotStages) & 1);
    const float* tile = reinterpret_cast<const float*>(tiles + st * stage_bytes + (tile_src(i) & 15));
    float* m = mrow + st * R;
    for (int r = warp; r < n; r += nw) {   // m[t] once per frame for the whole CTA
      const float mx = warp_row_max(tile + static_cast<int64_t>(r) * V1, V1, lane);
      if (lane == 0) m[r] = mx;
    }
    __syncthreads();   // m of this tile is published; every warp is done with tile i - 1's stage
    if (tid == 0 && i >= 1 && i - 1 + kSpotStages < ntiles) issue(i - 1 + kSpotStages);
    if (!active) continue;
    for (int r = 0; r < n; ++r) {
      const int t = fb + f0 + i * R + r;
      const float* row = tile + static_cast<int64_t>(r) * V1;
      const float mt = m[r];
      // frame t - 1 of lane - 1's last two states: the s - 1 / s - 2 predecessors of this lane's first two
      float pv3 = __shfl_up_sync(kFull, v[3], 1), pv2 = __shfl_up_sync(kFull, v[2], 1);
      const int pa3 = __shfl_up_sync(kFull, a[3], 1), pa2 = __shfl_up_sync(kFull, a[2], 1);
      if (lane == 0) pv3 = pv2 = -INFINITY;
      float nv[4];
      int na[4];
      if (isnan(mt)) {   // a barrier: no path crosses a frame whose row holds a NaN
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          nv[j] = -INFINITY;
          na[j] = t;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float best = v[j];
          int start = a[j];
          const float c1 = j >= 1 ? v[j - 1] : pv3;
          const int a1 = j >= 1 ? a[j - 1] : pa3;
          if (c1 > best) { best = c1; start = a1; }
          if (skip[j]) {
            const float c2 = j >= 2 ? v[j - 2] : (j == 1 ? pv3 : pv2);
            const int a2 = j >= 2 ? a[j - 2] : (j == 1 ? pa3 : pa2);
            if (c2 > best) { best = c2; start = a2; }
          }
          if (j == 0 && lane == 0 && 0.f > best) { best = 0.f; start = t; }   // state 0: a fresh path starts at t
          nv[j] = live[j] ? (row[lab[j]] - mt) + best : -INFINITY;
          na[j] = start;
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] = nv[j];
        a[j] = na[j];
      }
      // the end state's score and start, then the detection scan (every lane keeps the same pending detection)
      const float e_mine = e_slot == 0 ? v[0] : e_slot == 1 ? v[1] : e_slot == 2 ? v[2] : v[3];
      const int s_mine = e_slot == 0 ? a[0] : e_slot == 1 ? a[1] : e_slot == 2 ? a[2] : a[3];
      const float E = __shfl_sync(kFull, e_mine, e_lane);
      const int Es = __shfl_sync(kFull, s_mine, e_lane);
      if (E >= tau) {
        if (has && Es < p_end) {   // overlaps the pending detection: replace it only when strictly better
          if (E > p_score) { p_start = Es; p_end = t + 1; p_score = E; }
        } else {
          if (has) emit();
          has = 1;
          p_start = Es;
          p_end = t + 1;
          p_score = E;
        }
      }
    }
  }
  if (k >= K) return;
  if (has) {
    // a call without finish emits the pending detection early when no live path (finite score) starts before its end: a
    // later candidate starts at or after it, so it can no longer be replaced, only follow
    bool blocked = false;
    if (resume && io.finish[b] == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) blocked |= v[j] > -INFINITY && a[j] < p_end;
    }
    if (!__any_sync(kFull, blocked)) {
      emit();
      has = 0;
    }
  }
  if (resume) {
    if (active) {
      if (lane < L) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          rec_v[j * L + lane] = v[j];
          rec_a[j * L + lane] = a[j];
        }
      }
      if (lane == 0) {
        rec->has = has;
        rec->p_start = p_start;
        rec->p_end = p_end;
        rec->p_score = p_score;
        rec->total = total + (count - base);
        det_count[static_cast<int64_t>(b) * K + k] = min(count, max_det);
      }
    }
    if (lane == 0 && io.pend_start) {
      const int64_t p = static_cast<int64_t>(b) * K + k;
      io.pend_start[p] = has ? p_start : -1;
      io.pend_end[p] = has ? p_end : -1;
      io.pend_score[p] = has ? p_score : active ? -INFINITY : __int_as_float(0x7fc00000);
    }
    return;
  }
  if (lane == 0) det_count[static_cast<int64_t>(b) * K + k] = active ? count : 0;
  const float fill = active ? -INFINITY : __int_as_float(0x7fc00000);
  for (int i = (active ? min(count, max_det) : 0) + lane; i < max_det; i += 32) {
    det_start[row0 + i] = -1;
    det_end[row0 + i] = -1;
    det_score[row0 + i] = fill;
  }
}

__global__ void spot_state_init_kernel(uint8_t* state, int64_t n, int L, int64_t record) {
  const int64_t r = blockIdx.x;
  if (r >= n) return;
  SpotRecord* rec = reinterpret_cast<SpotRecord*>(state + r * record);
  float* v = reinterpret_cast<float*>(rec + 1);
  int* a = reinterpret_cast<int*>(v + 4 * L);
  for (int i = threadIdx.x; i < 4 * L; i += blockDim.x) {
    v[i] = -INFINITY;
    a[i] = 0;
  }
  if (threadIdx.x == 0) *rec = SpotRecord{0, 0, 0, 0, 0.f, {0, 0, 0}};
}

}  // namespace

int64_t ctc_spot_record_bytes(int Umax) {
  return static_cast<int64_t>(sizeof(SpotRecord)) + 8 * 4 * static_cast<int64_t>(spot_record_lanes(Umax));
}

void launch_ctc_spot_state_init(uint8_t* state, int64_t n, int Umax, cudaStream_t s) {
  if (n > 0) spot_state_init_kernel<<<static_cast<unsigned>(n), 128, 0, s>>>(state, n, spot_record_lanes(Umax), ctc_spot_record_bytes(Umax));
}

int ctc_spot_plan(int V1, int* rows, int* smem_bytes) {
  int dev = 0, cap = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return -1;
  const int R = std::min(std::max(kSpotTileBytes / (V1 * 4), 1), kSpotMaxRows);
  const int64_t stage = (static_cast<int64_t>(R) * V1 * 4 + 32 + 127) / 128 * 128;
  const int64_t smem = kSpotHeader + kSpotStages * stage;
  if (smem > cap) return 1;
  *rows = R;
  *smem_bytes = static_cast<int>(smem);
  return 0;
}

int launch_ctc_spot(const float* log_probs, const SpotResume& io, const int* keywords, const int* keyword_len, int B, int T, int V1, int K,
                    int Umax, float log_theta, int max_det, int warps, int* det_start, int* det_end, float* det_score, int* det_count,
                    cudaStream_t s) {
  static PerDeviceOnce attr_once;
  int R = 0, smem = 0;
  const int rc = ctc_spot_plan(V1, &R, &smem);
  if (rc != 0) return rc;
  if (attr_once.first()) {
    int dev = 0, cap = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (cudaFuncSetAttribute(ctc_spot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap) != cudaSuccess) return -1;
  }
  if (warps <= 0) warps = std::min(kSpotWarps, K);
  const int stage_bytes = (smem - kSpotHeader) / kSpotStages;
  const dim3 grid((K + warps - 1) / warps, B);
  ctc_spot_kernel<<<grid, 32 * warps, smem, s>>>(log_probs, io, keywords, keyword_len, T, V1, K, Umax, log_theta, max_det, R,
                                                 stage_bytes, det_start, det_end, det_score, det_count);
  return 0;
}

}  // namespace gam
