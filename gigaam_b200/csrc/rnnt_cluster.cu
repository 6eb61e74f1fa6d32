// RNN-T greedy decode, cluster-resident variant (gigaam/decoding.py:128-207, gigaam/decoder.py:24-102).
//
// The serial recurrence per utterance (see rnnt.cu) is latency bound; what made the one-CTA-per-utterance kernel
// slow was streaming W_hh (1.6 MB fp32) and W_p through one SM's L2 port on every emission.  Here a thread-block
// cluster of 16 CTAs keeps the weights RESIDENT in distributed shared memory: CTA c owns hidden units
// [c*H/16, (c+1)*H/16) -> its 4 gate rows of W_hh (80 x 320 fp32), its rows of W_p (20 x 320) and its slice of the
// output classes (rows of W_o: as many as fit next to the recurrent weights, the rest is prefetched from L2 into
// registers at the top of every joint phase).  A cluster decodes a group of up to 8 utterances in lock-step
// (utterances are independent; every CTA derives the same control flow from the same exchanged argmax results):
//   LSTM phase  (only utterances that just emitted): own gate rows . h  -> c', h' slice -> DSMEM all-to-all
//   pred phase  : own rows of W_p . h'                                  -> DSMEM all-to-all
//   joint phase : hid = relu(W_e e_t + b_e + pg);  own slice of classes -> local (max, argmax) -> DSMEM all-to-all
//
// Why the kernel is built this way (tools/rnnt_phase_probe.py times its phases):
//  * cg::cluster.sync() compiles to MEMBAR.ALL.GPU + ERRBAR + cluster barrier + CCTL.IVALL (~1 000 cycles, and it
//    drains every prefetch).  The round loop therefore has NO cluster barrier: every exchange is a set of 16-byte
//    st.async stores whose arrival is counted on an mbarrier of the RECEIVING CTA (two barriers per exchange type,
//    alternating, so bytes of consecutive exchanges can never mix); a CTA waits only on its own barriers.
//  * scalar control flow replicated in 16 warps costs 4x its single-warp time (4 warps per scheduler): the per-utterance
//    state lives in shared memory and ONE warp (one lane per utterance) takes the decision for the CTA.
//  * an H100 can keep only a few clusters of 16 CTAs resident, so 32 utterances in groups of 4 need two passes: groups hold
//    up to 8 utterances (two float4 halves), all state vectors are utterance-interleaved ([half][unit] -> float4), a
//    weight is read from shared memory once per phase for all of them, and exchanges are 16-byte stores.
//  * the prediction-network state is double-buffered by a cluster-wide parity that flips on every LSTM round;
//    utterances that do not step in that round carry their state over inside the same float4.
// All arithmetic is fp32 as in the reference head.
//
// Decision contract: the label of a joint row is what torch gives for log_softmax(row).argmax(-1) (gigaam/decoder.py:47,
// gigaam/decoding.py:162): on a row whose maximum is finite, the first maximal index; if any logit is NaN or +inf, or
// no logit exceeds -inf, label 0 (torch's log_softmax turns such a row all-NaN, and argmax of all-NaN is 0).  The label
// is therefore always in [0, V1).  A NaN or +inf logit enters the argmax as (+inf, index -1), which wins every later
// compare and every merge (equal values: lower index); warp 0 maps index -1 ("non-finite seen") and the empty index
// 0x7fffffff ("no winner") to 0.  hid keeps NaN as relu(NaN) = NaN does.
//
// Scored instantiation (SCORED, gam_rnnt_greedy_scored): every decision row also yields l = log_softmax(row)[label] =
// -log sum_c exp(z_c - z_max) (NaN where the label is 0 by the non-finite rule).  Each warp keeps, beside its running
// (max, argmax), the sum of exp(z - max) over its classes, rescaled when the max moves; warp 0 folds the 16 warp partials
// and, after the best-value exchange (which then carries that sum as a third float per utterance-half), the 16 CTA
// partials.  Both folds run in an order fixed by the warp / CTA index alone (4 runs of 4 in index order, then
// (0 + 1) + (2 + 3)), whatever the group width, so an utterance's scores do not depend on the batch it is decoded in.
// Warp 0 writes l on emission and sums it (fp64) over the utterance's decision rows.  The unscored instantiation
// compiles none of this.
//
// Boosted instantiation (BOOST, gam_rnnt_greedy_boost): utterance u is in state q_u of a boost graph, and the argmax runs
// over fp32(z_c + bonus[q_u, c]) (blank: + 0) with the same first-index and non-finite rules.  Each CTA keeps its own class
// slice of bonus[q_u] for every utterance of the group in shared memory (taken out of the W_o rows).  After an emission
// warp kStage0 moves q_u along next[q_u, label] (an entry outside [0, S): state 0) and warps kStage0.. restage the slices of
// the utterances that emitted; those warps have no work in the LSTM and prediction phases that every emission triggers, so
// the table loads run beside them.  When scored, l stays the model's own log_softmax(z)[label]: the lanes keep the
// log-sum-exp of z on its own running maximum, the argmax carries the winner's unboosted z, and the best-value exchange
// carries both, so l = -(log sum_c exp(z_c - z_max) - (z_label - z_max)), which is -log sum bit for bit with zero bonuses.
// q_u is stored in the record's boost_state.
#include <cooperative_groups.h>

#include <cstdlib>

#include "kernels.h"
#include "ptx.cuh"

namespace cg = cooperative_groups;

namespace gam {
namespace {

constexpr int kCl = 16;           // CTAs per cluster
constexpr int kMaxU = 8;          // utterances decoded in lock-step per cluster (two float4 halves)
constexpr int kH = 320;
constexpr int kHS = kH / kCl;     // hidden units owned per CTA (20)
constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kWhhP = 324;        // W_hh row pitch (words), 4 mod 32: (8 rows x 4 k-lanes) warps read conflict-free
constexpr int kWpP = 336;         // W_p row pitch, 16 mod 32: (2 rows x 16 k-lanes) warps read conflict-free
constexpr int kWoPitch = kH + 1;  // W_o row pitch: conflict-free 4-byte row walks
constexpr int kCB = 4;            // classes accumulated together per warp (one hid read serves all of them)
constexpr int kGP = 2;            // L2-resident class rows a warp prefetches into registers per round

struct RnntClParams {
  const float* encproj;    // [B*T, H]
  const float* emb_gates;  // [V1, 4H]
  const float* whhT;       // [H, 4H]  (W_hh^T)
  const float* wpT;        // [H, H]   (W_p^T)
  const float* bp;
  const float* wo;         // [V1, H]
  const float* bo;
  int B, T, V1, blank, max_symbols, num_groups, nu;   // nu <= 4 * NH utterances per group
  int rows_smem;           // class rows of W_o resident in shared memory per CTA
  int cls_pad;             // floats reserved for the bias slice
  GreedyIo io;             // outputs and stream ranges (kernels.h); io.state == NULL: a fresh call
  BoostGraph boost;        // read by the boosted instantiation only
};

// per-utterance decoding state (gigaam/decoding.py:150-205), owned by warp 0 of every CTA (identical in all of them)
struct Ctl {
  int t[kMaxU], nsym[kMaxU], cnt[kMaxU], label[kMaxU], L[kMaxU], need[kMaxU];
  int act_m, run_m, moved_m, emit_m;   // bit u: still decoding / needs an LSTM step / frame advanced / emitted a token
};

template <int NH>
struct Smem {
  float whh[4 * kHS][kWhhP];      // rows: gate g, unit j  ->  g*kHS + j
  float wp[kHS][kWpP];
  float4 h4[2][NH][kH];           // prediction-network state h, [parity][half][unit] -> 4 utterances (replicated per CTA)
  float4 pg4[NH][kH];             // W_p h' + b_p
  float4 hid4[NH][kH];            // relu(enc_proj[t] + pg)
  float4 hnew4[NH][kHS];          // own slice of the next state, staged for the 16-byte all-to-all
  float c[2][4 * NH][kHS];        // cell state of the own units, same parity as h4
  float gates[4 * NH][4 * kHS];
  float4 best_v[2][kCl][NH];      // per-CTA partial argmax, [exchange parity][source CTA]
  int4 best_i[2][kCl][NH];
  float wbest_v[kWarps][4 * NH];
  int wbest_i[kWarps][4 * NH];
  float4 my_v[NH];
  int4 my_i[NH];
  Ctl ctl;
  uint64_t bar_h[2], bar_pg[2], bar_best[2];   // arrival of the three all-to-all exchanges (alternating pairs)
  // followed by: [ScoreSmem<NH> if SCORED]; [BoostSmem<NH> if BOOST]; [BoostScoreSmem<NH> if BOOST and SCORED];
  // float bo[cls_pad]; [float bonus[4 NH][cls_pad] if BOOST]; float wo[rows_smem][kWoPitch];
};

// what the scored instantiation adds after Smem
template <int NH>
struct ScoreSmem {
  float4 best_s[2][kCl][NH];      // per-CTA partial sum of exp(z - CTA max), exchanged beside best_v / best_i
  float wbest_s[kWarps][4 * NH];
  float4 my_s[NH];
  double path[kMaxU];             // sum of l over the decision rows so far (warp 0, lane u)
  int rows[kMaxU];
};

// what the boosted instantiation adds
template <int NH>
struct BoostSmem {
  int q[kMaxU];                   // boost graph state per utterance (warp kStage0, lane u)
};
// ... and, when also scored: the maximum of the unboosted z and the winner's unboosted z beside the boosted argmax
template <int NH>
struct BoostScoreSmem {
  float4 best_m[2][kCl][NH], best_z[2][kCl][NH];
  float wbest_m[kWarps][4 * NH], wbest_z[kWarps][4 * NH];
  float4 my_m[NH], my_z[NH];
};

// Bytes one CTA receives per best-value exchange: one 16-byte store per utterance-half from each CTA of the cluster for
// every field of the payload (best_v, best_i and, when scored, best_s; boosted and scored, also best_m and best_z).  The
// expect-tx count of bar_best is this value, and the receive buffers of one parity are sized from the same constant, so the
// two cannot disagree.
template <int NH, bool SCORED, bool BOOST = false>
constexpr uint32_t best_exchange_bytes() { return kCl * NH * (SCORED ? (BOOST ? 5 : 3) : 2) * 16; }
static_assert(sizeof(Smem<1>::best_v[0]) + sizeof(Smem<1>::best_i[0]) == best_exchange_bytes<1, false>(), "best exchange payload");
static_assert(sizeof(Smem<2>::best_v[0]) + sizeof(Smem<2>::best_i[0]) == best_exchange_bytes<2, false>(), "best exchange payload");
static_assert(sizeof(Smem<1>::best_v[0]) + sizeof(Smem<1>::best_i[0]) + sizeof(ScoreSmem<1>::best_s[0]) ==
              best_exchange_bytes<1, true>(), "scored best exchange payload");
static_assert(sizeof(Smem<2>::best_v[0]) + sizeof(Smem<2>::best_i[0]) + sizeof(ScoreSmem<2>::best_s[0]) ==
              best_exchange_bytes<2, true>(), "scored best exchange payload");
static_assert(sizeof(Smem<2>::best_v[0]) + sizeof(Smem<2>::best_i[0]) + sizeof(ScoreSmem<2>::best_s[0]) +
              sizeof(BoostScoreSmem<2>::best_m[0]) + sizeof(BoostScoreSmem<2>::best_z[0]) == best_exchange_bytes<2, true, true>(),
              "boosted scored best exchange payload");
static_assert(sizeof(float4) == 16 && sizeof(int4) == 16, "push16 moves one float4 / int4");

template <int NH, bool SCORED, bool BOOST = false>
constexpr int fixed_smem_bytes() {
  return static_cast<int>(sizeof(Smem<NH>) + (SCORED ? sizeof(ScoreSmem<NH>) : 0) + (BOOST ? sizeof(BoostSmem<NH>) : 0) +
                          (BOOST && SCORED ? sizeof(BoostScoreSmem<NH>) : 0));
}
static_assert(sizeof(ScoreSmem<1>) % 16 == 0 && sizeof(ScoreSmem<2>) % 16 == 0 && sizeof(BoostSmem<2>) % 16 == 0,
              "the shared-memory parts stay 16-byte aligned");
// every byte of shared memory in front of the W_o rows: the fixed parts, the bias slice and (boosted) the bonus slices
template <int NH, bool SCORED, bool BOOST>
constexpr int smem_before_rows(int cls_pad) { return fixed_smem_bytes<NH, SCORED, BOOST>() + cls_pad * 4 * (1 + (BOOST ? 4 * NH : 0)); }

__device__ __forceinline__ float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float comp(const float4& v, int u) { return u == 0 ? v.x : (u == 1 ? v.y : (u == 2 ? v.z : v.w)); }
__device__ __forceinline__ void set_comp(float4& v, int u, float x) {
  if (u == 0) v.x = x; else if (u == 1) v.y = x; else if (u == 2) v.z = x; else v.w = x;
}

// sum of v over the warp; returns the total of component u = (lane >> 3) & 3  (6 shuffles instead of 20)
__device__ __forceinline__ float reduce4(const float4 v, int lane) {
  const bool hi = (lane & 16) != 0;
  float k0 = hi ? v.z : v.x, k1 = hi ? v.w : v.y;
  k0 += __shfl_xor_sync(0xffffffffu, hi ? v.x : v.z, 16);
  k1 += __shfl_xor_sync(0xffffffffu, hi ? v.y : v.w, 16);
  const bool mid = (lane & 8) != 0;
  float k = mid ? k1 : k0;
  k += __shfl_xor_sync(0xffffffffu, mid ? k0 : k1, 8);
  k += __shfl_xor_sync(0xffffffffu, k, 4);
  k += __shfl_xor_sync(0xffffffffu, k, 2);
  k += __shfl_xor_sync(0xffffffffu, k, 1);
  return k;
}

// relu that keeps NaN (torch.relu); fmaxf(x, 0) would turn NaN into 0
__device__ __forceinline__ float relu_nan(float x) { return x < 0.f ? 0.f : x; }

// running argmax over ascending classes: strict > keeps the first maximum; a NaN or +inf logit becomes (+inf, -1), the
// "non-finite seen" mark that no later logit replaces and that wins every merge
__device__ __forceinline__ void arg_update(float a, int cls, float& bv, int& bi) {
  if (!(a <= bv)) {
    const bool bad = !(a < INFINITY);
    bv = bad ? INFINITY : a;
    bi = bad ? -1 : cls;
  }
}

// boosted argmax update: the argmax of arg_update over a = z + b, carrying the winner's z (bz); when scored, the sum of
// exp(z - zm) over the finite z relative to their own running maximum zm, by arg_update_s's rule
template <bool SCORED>
__device__ __forceinline__ void arg_update_b(float z, float b, int cls, float& bv, int& bi, float& bz, float& zm, float& bs) {
  const float a = z + b;
  if (!(a <= bv)) {
    const bool bad = !(a < INFINITY);
    bv = bad ? INFINITY : a;
    bi = bad ? -1 : cls;
    bz = z;
  }
  if constexpr (SCORED) {
    if (!(z <= zm)) {
      const bool bad = !(z < INFINITY);
      if (!bad) bs = bs * expf(zm - z) + 1.f;
      zm = bad ? INFINITY : z;
    } else if (z > -INFINITY) {
      bs += expf(z - zm);
    }
  }
}

// arg_update plus, when scored, the running sum of exp(a - bv) over the finite logits (rescaled when bv moves; bv = -inf
// at the start gives 0 * 0 + 1).  After a NaN / +inf logit the sum is meaningless and l becomes NaN.
template <bool SCORED>
__device__ __forceinline__ void arg_update_s(float a, int cls, float& bv, int& bi, float& bs) {
  if constexpr (SCORED) {
    if (!(a <= bv)) {
      const bool bad = !(a < INFINITY);
      if (!bad) bs = bs * expf(bv - a) + 1.f;
      bv = bad ? INFINITY : a;
      bi = bad ? -1 : cls;
    } else if (a > -INFINITY) {
      bs += expf(a - bv);
    }
  } else {
    arg_update(a, cls, bv, bi);
  }
}

// scored fold of 16 partials (value v_k, sum s_k relative to v_k) to the sum relative to the maximum m: lane `lane` of
// utterance u = lane % nu folds partials 4 sub .. 4 sub + 3 (sub = lane / nu < 4), then (0 + 1) + (2 + 3) across subs.
// The order depends on the partial index alone, not on nu (4 or 8); the result is in the lanes of sub 0.
template <typename VS>
__device__ __forceinline__ float fold16(VS vs, float m, int nu, int lane) {
  const int sub = lane / nu;
  float acc = 0.f;
  if (sub < 4) {
#pragma unroll
    for (int k = 4 * sub; k < 4 * sub + 4; ++k) {
      float v, sk;
      vs(k, v, sk);
      if (v > -INFINITY) acc += sk * expf(v - m);
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, nu);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2 * nu);
  return acc;
}

__device__ __forceinline__ void fma4(float4& a, float w, const float4& h) {
  a.x = fmaf(w, h.x, a.x); a.y = fmaf(w, h.y, a.y); a.z = fmaf(w, h.z, a.z); a.w = fmaf(w, h.w, a.w);
}

// 16-byte counted store to the same shared-memory location (and barrier) in CTA `cta` of the cluster
__device__ __forceinline__ void push16(const void* local_dst, uint64_t* local_bar, uint32_t cta, uint32_t a, uint32_t b, uint32_t c,
                                       uint32_t d) {
  ptx::st_async_v4(ptx::mapa_u32(ptx::smem_u32(local_dst), cta), ptx::mapa_u32(ptx::smem_u32(local_bar), cta), a, b, c, d);
}
__device__ __forceinline__ void push16(const void* local_dst, uint64_t* local_bar, uint32_t cta, const float4& v) {
  push16(local_dst, local_bar, cta, __float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w));
}

// stream b's DecodeState, or NULL on a fresh call
__device__ __forceinline__ DecodeState* state_of(const RnntClParams& p, int b) {
  return p.io.state ? reinterpret_cast<DecodeState*>(p.io.state + b * p.io.stride) : nullptr;
}

#ifdef GAM_RNNT_DBG
// phase timing of cluster 0 / CTA 0 / thread 0 (tools/rnnt_phase_probe.py; never compiled into the shipped library)
__device__ long long g_rnnt_dbg[16];
#define DBG_T(i) do { if (dbg_on) { const long long t_now = clock64(); dbg_acc[i] += t_now - dbg_last; dbg_last = t_now; } } while (0)
#else
#define DBG_T(i) do { } while (0)
#endif

// NH: float4 halves of utterances per group (4 or 8 utterances).  GLOB: some class rows stay in L2 (large vocabularies);
// compiled out otherwise (the round loop is executed once per step by every warp; 16 KB less code).
// A resume call (p.io.state set, gam_rnnt_greedy_resume) starts a group from the DecodeState records of its utterances --
// control state, label, pending LSTM step, h, c and pg -- decodes frames [lo, hi) of each row and stores the state back.
// A fresh call starts from the constants of a fresh record (blank label, a pending step, zeros) and decodes [0, hi).  A chunk
// edge is a frame edge (nsym = 0), so decoding [0, L) in consecutive chunks runs the same operations on the same values as
// one fresh call.
template <int NH, bool GLOB, bool SCORED, bool BOOST>
__global__ void __launch_bounds__(kThreads, 1) rnnt_cluster_kernel(const RnntClParams p) {
  constexpr int NU = 4 * NH;
  using SM = Smem<NH>;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SM& s = *reinterpret_cast<SM*>(smem_raw);
  [[maybe_unused]] ScoreSmem<NH>& sc = *reinterpret_cast<ScoreSmem<NH>*>(smem_raw + sizeof(SM));
  float* s_bo = reinterpret_cast<float*>(smem_raw + fixed_smem_bytes<NH, SCORED, BOOST>());
  float* s_wo = s_bo + p.cls_pad;
  // boosted: q per utterance, the scored exchange fields and bonus[q_u] over the own classes ([u][cls_pad])
  [[maybe_unused]] int* s_q = nullptr;
  [[maybe_unused]] BoostScoreSmem<NH>* bss = nullptr;
  [[maybe_unused]] float* s_bon = nullptr;
  constexpr bool BS = BOOST && SCORED;
  if constexpr (BOOST) {
    constexpr int off = sizeof(SM) + (SCORED ? sizeof(ScoreSmem<NH>) : 0);
    s_q = reinterpret_cast<BoostSmem<NH>*>(smem_raw + off)->q;
    bss = reinterpret_cast<BoostScoreSmem<NH>*>(smem_raw + off + sizeof(BoostSmem<NH>));
    s_bon = s_wo;
    s_wo += NU * p.cls_pad;
  }
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cluster_id = blockIdx.x / kCl;
  const int num_clusters = gridDim.x / kCl;
  const int G = 4 * kH;
#ifdef GAM_RNNT_DBG
  const bool dbg_on = blockIdx.x == 0 && threadIdx.x == 0;
  long long dbg_acc[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  long long dbg_last = clock64();
#endif

  // ---- resident weight slices (once per kernel)
  for (int i = tid; i < 4 * kHS * kH; i += kThreads) {
    const int r = i / kH, k = i % kH;                    // r = g*kHS + j
    const int g = r / kHS, j = r % kHS;
    s.whh[r][k] = __ldg(p.whhT + static_cast<size_t>(k) * G + g * kH + rank * kHS + j);
  }
  for (int i = tid; i < kHS * kH; i += kThreads) {
    const int j = i / kH, k = i % kH;
    s.wp[j][k] = __ldg(p.wpT + static_cast<size_t>(k) * kH + rank * kHS + j);
  }
  const int cls_per = (p.V1 + kCl - 1) / kCl;
  const int cls0 = min(p.V1, rank * cls_per);
  const int ncls = min(p.V1, cls0 + cls_per) - cls0;       // classes owned by this CTA
  const int nsm = min(ncls, p.rows_smem);                  // ... of which resident in shared memory
  for (int i = tid; i < nsm * kH; i += kThreads) s_wo[(i / kH) * kWoPitch + i % kH] = __ldg(p.wo + static_cast<size_t>(cls0 + i / kH) * kH + i % kH);
  for (int i = tid; i < ncls; i += kThreads) s_bo[i] = __ldg(p.bo + cls0 + i);
  // LSTM-phase role of this thread: gate row lr_row, k-lane lq; lane q of a quad also finishes utterances q, q+4
  const int lq = lane & 3, lr_row = warp * 8 + (lane >> 2);
  const bool gate_thread = warp < 4 * kHS / 8;
  const size_t eg_off = gate_thread ? static_cast<size_t>((lr_row / kHS) * kH + rank * kHS + lr_row % kHS) : 0;
  // pred-phase role: row pj, k-lane pq (which is also the CTA this lane serves in the all-to-all)
  const int pq = lane & 15, pj = warp * 2 + (lane >> 4);
  const bool pred_thread = warp < kHS / 2;
  const float my_bp = pred_thread ? __ldg(p.bp + rank * kHS + pj) : 0.f;
  // boosted: warps kStage0.. (no LSTM or prediction role) keep the bonus slices; stage(m) loads bonus[q_u] over the own
  // classes for the utterances of mask m (blank: 0)
  constexpr int kStage0 = 4 * kHS / 8, kStageThreads = kThreads - 32 * kStage0;
  static_assert(kHS / 2 <= kStage0 && kStageThreads % 32 == 0, "the staging warps have no LSTM or prediction role");
  [[maybe_unused]] auto stage = [&](unsigned m) {
    for (int i = tid - 32 * kStage0; i < NU * ncls; i += kStageThreads) {
      const int u = i / ncls, c = i - u * ncls;
      if ((m >> u) & 1) {
        const int cls = cls0 + c;
        s_bon[u * p.cls_pad + c] = cls == p.blank ? 0.f : __ldg(p.boost.bonus + static_cast<size_t>(s_q[u]) * p.V1 + cls);
      }
    }
  };
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      ptx::mbar_init(&s.bar_h[i], 1);
      ptx::mbar_init(&s.bar_pg[i], 1);
      ptx::mbar_init(&s.bar_best[i], 1);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  uint32_t n_h = 0, n_pg = 0, n_b = 0;   // exchanges done so far (barrier = n & 1, phase parity = (n >> 1) & 1)
  constexpr uint32_t kStateBytes = kCl * kHS * NH * 16;
  constexpr uint32_t kBestBytes = best_exchange_bytes<NH, SCORED, BOOST>();

  for (int group = cluster_id; group < p.num_groups; group += num_clusters) {
    // warp 0 lane u: counts[b] when the call started, frame_base[b], and the current frame's sum of l and rows
    int r_cnt0 = 0, r_fb = 0;
    [[maybe_unused]] int r_frows = 0;
    [[maybe_unused]] double r_facc = 0.0;
    // ---- start of the group: control state (warp 0: lane u = utterance u), read from the DecodeState records on a resume
    // call; lanes without an utterance start inactive
    if (warp == 0) {
      int Lu = 0, t0 = 0, pend = 0;
      if (lane < kMaxU) {
        const int ug = group * p.nu + lane;
        int lbl = p.blank, rows = 0;
        double path = 0.0;
        if (lane < p.nu && lane < NU && ug < p.B) {
          const DecodeState* st = state_of(p, ug);
          t0 = st ? min(max(p.io.lo[ug], 0), p.T) : 0;
          Lu = min(max(p.io.hi[ug], t0), p.T);
          pend = 1;
          if (st) {
            lbl = st->label; pend = st->pending; path = st->path; rows = st->rows;
            r_cnt0 = p.io.counts[ug]; r_fb = p.io.frame_base[ug];
          }
        }
        s.ctl.t[lane] = t0; s.ctl.nsym[lane] = 0; s.ctl.cnt[lane] = r_cnt0; s.ctl.label[lane] = lbl;
        s.ctl.L[lane] = Lu; s.ctl.need[lane] = pend;
        if constexpr (SCORED) { sc.path[lane] = path; sc.rows[lane] = rows; }
      }
      // only the utterances with a pending step run the first LSTM round
      const unsigned am = __ballot_sync(0xffffffffu, Lu > t0), rm = __ballot_sync(0xffffffffu, Lu > t0 && pend != 0);
      if (lane == 0) { s.ctl.act_m = static_cast<int>(am); s.ctl.run_m = static_cast<int>(rm); s.ctl.moved_m = 0; s.ctl.emit_m = 0; }
    }
    // h, pg (all units, utterance-interleaved) and c (own units): from the records, or zero
    for (int i = tid; i < NH * kH; i += kThreads) {
      const int hh = i / kH, k = i % kH;
      float4 hv = make_float4(0.f, 0.f, 0.f, 0.f), gv = hv;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int u = 4 * hh + cc, ug = group * p.nu + u;
        const DecodeState* st = u < p.nu && ug < p.B ? state_of(p, ug) : nullptr;
        if (st) {
          set_comp(hv, cc, st->h[k]);
          set_comp(gv, cc, st->pg[k]);
        }
      }
      s.h4[0][hh][k] = hv;
      s.h4[1][hh][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      s.pg4[hh][k] = gv;
    }
    for (int i = tid; i < NU * kHS; i += kThreads) {
      const int u = i / kHS, j = i % kHS, ug = group * p.nu + u;
      const DecodeState* st = u < p.nu && ug < p.B ? state_of(p, ug) : nullptr;
      s.c[0][u][j] = st ? st->c[rank * kHS + j] : 0.f;
      s.c[1][u][j] = 0.f;
    }
    if constexpr (BOOST) {   // q from the records (a fresh record holds 0), then every utterance's bonus slice
      if (warp >= kStage0) {
        if (warp == kStage0 && lane < kMaxU) {
          const int ug = group * p.nu + lane;
          const DecodeState* st = lane < p.nu && lane < NU && ug < p.B ? state_of(p, ug) : nullptr;
          const int q = st ? st->boost_state : 0;
          s_q[lane] = q >= 0 && q < p.boost.n_states ? q : 0;
        }
        ptx::named_bar_sync<kStageThreads>(1);
        stage(0xffffffffu);
      }
    }
    __syncthreads();
    const int act0 = s.ctl.act_m;   // the utterances this call decodes (a resume call leaves the others' records and outputs)
    // encoder projection of the current frame (ep) and of the next one (epn): thread k < H keeps all utterances'
    // values in registers; a frame advance promotes epn and requests the frame after it
    float4 ep[NH], epn[NH];
    const float* ep_base = p.encproj + static_cast<size_t>(group * p.nu) * p.T * kH + (tid < kH ? tid : 0);
#pragma unroll
    for (int hh = 0; hh < NH; ++hh) {
      ep[hh] = make_float4(0.f, 0.f, 0.f, 0.f);
      epn[hh] = ep[hh];
      if (tid < kH) {
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) {
          const int u = 4 * hh + cc;
          const int Lu = s.ctl.L[u];
          const int t0 = s.ctl.t[u];
          if (Lu > t0) set_comp(ep[hh], cc, __ldg(ep_base + (static_cast<size_t>(u) * p.T + t0) * kH));
          if (Lu > t0 + 1) set_comp(epn[hh], cc, __ldg(ep_base + (static_cast<size_t>(u) * p.T + t0 + 1) * kH));
        }
      }
    }
    // embedding contribution to this thread's gates (row lr_row, utterances lq + 4 hh); reloaded after an emission
    float eg[NH];
#pragma unroll
    for (int hh = 0; hh < NH; ++hh) {
      eg[hh] = gate_thread ? __ldg(p.emb_gates + static_cast<size_t>(s.ctl.label[4 * hh + lq]) * G + eg_off) : 0.f;
    }
    int gb = 0;   // parity of the h4 / c buffer that holds the current prediction-network state of all utterances
    cluster.sync();   // every CTA's buffers and barriers are initialised before the first remote store can arrive
    DBG_T(6);

    while (true) {
      const int act_m = s.ctl.act_m, run_m = s.ctl.run_m;
      if (act_m == 0) break;
      DBG_T(9);
#ifdef GAM_RNNT_DBG
      dbg_acc[7] += 1;
      if (run_m != 0) dbg_acc[8] += 1;
#endif

      if (run_m != 0) {
        if (tid == 0) ptx::mbar_arrive_expect_tx(&s.bar_h[n_h & 1], kStateBytes);
        // ---------------- gates: warp = 8 own rows x 4 k-lanes (k = 16 i + 4 e + q)
        if (gate_thread) {
          const float* wrow = &s.whh[lr_row][lq];
          float4 a[NH];
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) a[hh] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
          for (int i = 0; i < kH / 16; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float w = wrow[16 * i + 4 * e];
#pragma unroll
              for (int hh = 0; hh < NH; ++hh) fma4(a[hh], w, s.h4[gb][hh][16 * i + 4 * e + lq]);
            }
          }
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) {
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
              a[hh].x += __shfl_xor_sync(0xffffffffu, a[hh].x, o); a[hh].y += __shfl_xor_sync(0xffffffffu, a[hh].y, o);
              a[hh].z += __shfl_xor_sync(0xffffffffu, a[hh].z, o); a[hh].w += __shfl_xor_sync(0xffffffffu, a[hh].w, o);
            }
            s.gates[4 * hh + lq][lr_row] = eg[hh] + comp(a[hh], lq);   // lane q of the quad finishes utterance 4 hh + q
          }
        }
        __syncthreads();
        DBG_T(0);
        if (tid < NU * kHS) {
          const int u = tid / kHS, j = tid % kHS;
          const float c_old = s.c[gb][u][j];
          float cn = c_old, hn = comp(s.h4[gb][u >> 2][rank * kHS + j], u & 3);   // utterances that do not step carry over
          if ((run_m >> u) & 1) {
            const float ig = sigm(s.gates[u][j]), fg = sigm(s.gates[u][kHS + j]);
            const float gg = tanhf(s.gates[u][2 * kHS + j]), og = sigm(s.gates[u][3 * kHS + j]);
            cn = fg * c_old + ig * gg;
            hn = og * tanhf(cn);
          }
          s.c[gb ^ 1][u][j] = cn;
          reinterpret_cast<float*>(&s.hnew4[u >> 2][j])[u & 3] = hn;
        }
        __syncthreads();
        for (int i = tid; i < kCl * NH * kHS; i += kThreads) {   // 16-byte counted stores: (CTA, half, unit)
          const int cta = i / (NH * kHS), hh = (i / kHS) % NH, j = i % kHS;
          push16(&s.h4[gb ^ 1][hh][rank * kHS + j], &s.bar_h[n_h & 1], cta, s.hnew4[hh][j]);
        }
        DBG_T(1);
        if (pred_thread) ptx::mbar_wait(&s.bar_h[n_h & 1], (n_h >> 1) & 1);
        ++n_h;
        DBG_T(2);
        // ---------------- prediction projection: own rows of W_p on the new state (warp = 2 rows x 16 k-lanes)
        if (tid == 0) ptx::mbar_arrive_expect_tx(&s.bar_pg[n_pg & 1], kStateBytes);
        if (pred_thread) {
          const float* wrow = &s.wp[pj][pq];
          float4 a[NH];
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) a[hh] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int i = 0; i < kH / 64; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float w = wrow[64 * i + 16 * e];
#pragma unroll
              for (int hh = 0; hh < NH; ++hh) fma4(a[hh], w, s.h4[gb ^ 1][hh][64 * i + 16 * e + pq]);
            }
          }
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) {
#pragma unroll
            for (int o = 1; o <= 8; o <<= 1) {
              a[hh].x += __shfl_xor_sync(0xffffffffu, a[hh].x, o); a[hh].y += __shfl_xor_sync(0xffffffffu, a[hh].y, o);
              a[hh].z += __shfl_xor_sync(0xffffffffu, a[hh].z, o); a[hh].w += __shfl_xor_sync(0xffffffffu, a[hh].w, o);
            }
            const float4 old = s.pg4[hh][rank * kHS + pj];
            const int rm = run_m >> (4 * hh);
            const float4 v = make_float4((rm & 1) ? my_bp + a[hh].x : old.x, (rm & 2) ? my_bp + a[hh].y : old.y,
                                         (rm & 4) ? my_bp + a[hh].z : old.z, (rm & 8) ? my_bp + a[hh].w : old.w);
            push16(&s.pg4[hh][rank * kHS + pj], &s.bar_pg[n_pg & 1], pq, v);   // lane q of the row's 16 serves CTA q
          }
        }
        DBG_T(3);
        if (pred_thread) ptx::mbar_wait(&s.bar_pg[n_pg & 1], (n_pg >> 1) & 1);   // warps 0-9 also build hid4 below
        ++n_pg;
        gb ^= 1;
        DBG_T(2);
      }

      // ---------------- joint: hid = relu(enc_proj[t] + pg), own class slice, local argmax
      if (tid == 0) ptx::mbar_arrive_expect_tx(&s.bar_best[n_b & 1], kBestBytes);
      // class rows that do not fit in shared memory: issue their L2 loads now, consume them after the smem rows
      [[maybe_unused]] float wg[kGP][kH / 32];
      [[maybe_unused]] int gcls[kGP];
      if constexpr (GLOB) {
#pragma unroll
        for (int gi = 0; gi < kGP; ++gi) {
          const int lr = nsm + ((warp - nsm) & (kWarps - 1)) + kWarps * gi;   // this warp's gi-th row at or after nsm
          gcls[gi] = lr < ncls ? lr : -1;
          if (gcls[gi] >= 0) {
            const float* w = p.wo + static_cast<size_t>(cls0 + lr) * kH;
#pragma unroll
            for (int kk = 0; kk < kH / 32; ++kk) wg[gi][kk] = __ldg(w + lane + 32 * kk);
          }
        }
      }
      if (tid < kH) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
          const float4 g4 = s.pg4[hh][tid];
          const int am = act_m >> (4 * hh);
          s.hid4[hh][tid] = make_float4((am & 1) ? relu_nan(ep[hh].x + g4.x) : 0.f, (am & 2) ? relu_nan(ep[hh].y + g4.y) : 0.f,
                                        (am & 4) ? relu_nan(ep[hh].z + g4.z) : 0.f, (am & 8) ? relu_nan(ep[hh].w + g4.w) : 0.f);
        }
      }
      __syncthreads();
      DBG_T(13);
      const int myu = (lane >> 3) & 3;       // the utterance (within a half) whose logits this lane ends up holding
      float bv[NH];
      int bi[NH];
      [[maybe_unused]] float bs[NH];
      [[maybe_unused]] float bz[NH], zm[NH];   // boosted: the winner's unboosted z; when scored, the running max of z
#pragma unroll
      for (int hh = 0; hh < NH; ++hh) { bv[hh] = -INFINITY; bi[hh] = 0x7fffffff; bs[hh] = 0.f; }
      if constexpr (BOOST) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) { bz[hh] = 0.f; zm[hh] = -INFINITY; }
      }
      [[maybe_unused]] const float* bon = s_bon + myu * p.cls_pad;   // bonus of utterance 4 hh + myu at bon[4 hh cls_pad + lr]
      // shared-memory rows: local rows warp, warp+16, ... (ascending, so the first maximum wins as in torch.argmax)
      for (int lr0 = warp; lr0 < nsm; lr0 += kWarps * kCB) {
        float4 acc[kCB][NH];
#pragma unroll
        for (int c = 0; c < kCB; ++c)
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) acc[c][hh] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int kk = 0; kk < kH / 32; ++kk) {
          const int k = lane + 32 * kk;
          float4 hv[NH];
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) hv[hh] = s.hid4[hh][k];
#pragma unroll
          for (int c = 0; c < kCB; ++c)
            if (lr0 + kWarps * c < nsm) {
              const float w = s_wo[(lr0 + kWarps * c) * kWoPitch + k];
#pragma unroll
              for (int hh = 0; hh < NH; ++hh) fma4(acc[c][hh], w, hv[hh]);
            }
        }
#pragma unroll
        for (int c = 0; c < kCB; ++c) {
          const int lr = lr0 + kWarps * c;
          if (lr < nsm) {
#pragma unroll
            for (int hh = 0; hh < NH; ++hh) {
              if constexpr (BOOST)
                arg_update_b<SCORED>(reduce4(acc[c][hh], lane) + s_bo[lr], bon[4 * hh * p.cls_pad + lr], cls0 + lr, bv[hh], bi[hh],
                                     bz[hh], zm[hh], bs[hh]);
              else
                arg_update_s<SCORED>(reduce4(acc[c][hh], lane) + s_bo[lr], cls0 + lr, bv[hh], bi[hh], bs[hh]);
            }
          }
        }
      }
      // L2 rows (registers), then anything beyond the prefetch depth straight from L2
      if constexpr (GLOB) {
#pragma unroll
      for (int gi = 0; gi < kGP; ++gi) {
        if (gcls[gi] >= 0) {
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int kk = 0; kk < kH / 32; ++kk) fma4(acc, wg[gi][kk], s.hid4[hh][lane + 32 * kk]);
            if constexpr (BOOST)
              arg_update_b<SCORED>(reduce4(acc, lane) + s_bo[gcls[gi]], bon[4 * hh * p.cls_pad + gcls[gi]], cls0 + gcls[gi], bv[hh],
                                   bi[hh], bz[hh], zm[hh], bs[hh]);
            else
              arg_update_s<SCORED>(reduce4(acc, lane) + s_bo[gcls[gi]], cls0 + gcls[gi], bv[hh], bi[hh], bs[hh]);
          }
        }
      }
      for (int lr = nsm + ((warp - nsm) & (kWarps - 1)) + kWarps * kGP; lr < ncls; lr += kWarps) {
        const float* w = p.wo + static_cast<size_t>(cls0 + lr) * kH;
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int kk = 0; kk < kH / 32; ++kk) fma4(acc, __ldg(w + lane + 32 * kk), s.hid4[hh][lane + 32 * kk]);
          if constexpr (BOOST)
            arg_update_b<SCORED>(reduce4(acc, lane) + s_bo[lr], bon[4 * hh * p.cls_pad + lr], cls0 + lr, bv[hh], bi[hh], bz[hh], zm[hh],
                                 bs[hh]);
          else
            arg_update_s<SCORED>(reduce4(acc, lane) + s_bo[lr], cls0 + lr, bv[hh], bi[hh], bs[hh]);
        }
      }
      }
      DBG_T(14);
      if ((lane & 7) == 0) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) { s.wbest_v[warp][4 * hh + myu] = bv[hh]; s.wbest_i[warp][4 * hh + myu] = bi[hh]; }
        if constexpr (SCORED) {
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) sc.wbest_s[warp][4 * hh + myu] = bs[hh];
        }
        if constexpr (BS) {
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) { bss->wbest_m[warp][4 * hh + myu] = zm[hh]; bss->wbest_z[warp][4 * hh + myu] = bz[hh]; }
        }
      }
      __syncthreads();
      DBG_T(15);

      // ---------------- warp 0: CTA argmax -> all-to-all -> decision (lane = utterance u + NU * sub-lane)
      if (warp == 0) {
        constexpr int kSub = 32 / NU;
        const int u = lane % NU, sub = lane / NU;
        const int par = n_b & 1;
        float v0 = -INFINITY;
        int i0 = 0x7fffffff;
        [[maybe_unused]] float z0 = 0.f, zmax = -INFINITY;   // boosted and scored: the winner's z and the maximum of z
        for (int w = sub; w < kWarps; w += kSub) {
          const float v = s.wbest_v[w][u];
          const int i = s.wbest_i[w][u];
          if (v > v0 || (v == v0 && i < i0)) {
            v0 = v; i0 = i;
            if constexpr (BS) z0 = bss->wbest_z[w][u];
          }
          if constexpr (BS) { const float m = bss->wbest_m[w][u]; if (m > zmax) zmax = m; }
        }
#pragma unroll
        for (int o = NU; o < 32; o <<= 1) {
          const float v = __shfl_xor_sync(0xffffffffu, v0, o);
          const int i = __shfl_xor_sync(0xffffffffu, i0, o);
          if constexpr (BS) {
            const float z = __shfl_xor_sync(0xffffffffu, z0, o), m = __shfl_xor_sync(0xffffffffu, zmax, o);
            if (v > v0 || (v == v0 && i < i0)) z0 = z;
            if (m > zmax) zmax = m;
          }
          if (v > v0 || (v == v0 && i < i0)) { v0 = v; i0 = i; }
        }
        if (lane < NU) { reinterpret_cast<float*>(s.my_v)[u] = v0; reinterpret_cast<int*>(s.my_i)[u] = i0; }
        if constexpr (BS) {   // the sum relative to the maximum of the unboosted z
          const float cs = fold16([&](int w, float& v, float& sk) { v = bss->wbest_m[w][u]; sk = sc.wbest_s[w][u]; }, zmax, NU, lane);
          if (lane < NU) {
            reinterpret_cast<float*>(sc.my_s)[u] = cs;
            reinterpret_cast<float*>(bss->my_m)[u] = zmax;
            reinterpret_cast<float*>(bss->my_z)[u] = z0;
          }
        } else if constexpr (SCORED) {   // the CTA's sum relative to its maximum v0 (every lane of utterance u holds v0)
          const float cs = fold16([&](int w, float& v, float& sk) { v = s.wbest_v[w][u]; sk = sc.wbest_s[w][u]; }, v0, NU, lane);
          if (lane < NU) reinterpret_cast<float*>(sc.my_s)[u] = cs;
        }
        __syncwarp();
        if (lane < kCl) {   // lane = destination CTA; one 16-byte store per field and half (best_exchange_bytes)
#pragma unroll
          for (int hh = 0; hh < NH; ++hh) {
            const int4 ii = s.my_i[hh];
            push16(&s.best_v[par][rank][hh], &s.bar_best[par], lane, s.my_v[hh]);
            push16(&s.best_i[par][rank][hh], &s.bar_best[par], lane, static_cast<uint32_t>(ii.x), static_cast<uint32_t>(ii.y),
                   static_cast<uint32_t>(ii.z), static_cast<uint32_t>(ii.w));
            if constexpr (SCORED) push16(&sc.best_s[par][rank][hh], &s.bar_best[par], lane, sc.my_s[hh]);
            if constexpr (BS) {
              push16(&bss->best_m[par][rank][hh], &s.bar_best[par], lane, bss->my_m[hh]);
              push16(&bss->best_z[par][rank][hh], &s.bar_best[par], lane, bss->my_z[hh]);
            }
          }
        }
        DBG_T(4);
        ptx::mbar_wait(&s.bar_best[par], (n_b >> 1) & 1);
        DBG_T(5);
        v0 = -INFINITY;
        i0 = 0x7fffffff;
        if constexpr (BS) { z0 = 0.f; zmax = -INFINITY; }
        for (int r = sub; r < kCl; r += kSub) {   // source CTAs ascend with the class index
          const float v = reinterpret_cast<const float*>(&s.best_v[par][r][0])[u];
          const int i = reinterpret_cast<const int*>(&s.best_i[par][r][0])[u];
          if (v > v0 || (v == v0 && i < i0)) {
            v0 = v; i0 = i;
            if constexpr (BS) z0 = reinterpret_cast<const float*>(&bss->best_z[par][r][0])[u];
          }
          if constexpr (BS) { const float m = reinterpret_cast<const float*>(&bss->best_m[par][r][0])[u]; if (m > zmax) zmax = m; }
        }
#pragma unroll
        for (int o = NU; o < 32; o <<= 1) {
          const float v = __shfl_xor_sync(0xffffffffu, v0, o);
          const int i = __shfl_xor_sync(0xffffffffu, i0, o);
          if constexpr (BS) {
            const float z = __shfl_xor_sync(0xffffffffu, z0, o), m = __shfl_xor_sync(0xffffffffu, zmax, o);
            if (v > v0 || (v == v0 && i < i0)) z0 = z;
            if (m > zmax) zmax = m;
          }
          if (v > v0 || (v == v0 && i < i0)) { v0 = v; i0 = i; }
        }
        DBG_T(10);
        // "non-finite seen" (-1) and "no winner" (0x7fffffff: every logit -inf) give label 0, as torch's argmax of an
        // all-NaN log_softmax row; the label that indexes emb_gates below is in [0, V1) by construction
        const int lab = (i0 < 0 || i0 >= p.V1) ? 0 : i0;
        [[maybe_unused]] float lp = 0.f;
        if constexpr (BS) {   // l of the unboosted row; -(log ts - 0) is -log ts bit for bit when the winner is the maximum
          const float ts = fold16([&](int r, float& v, float& sk) {
            v = reinterpret_cast<const float*>(&bss->best_m[par][r][0])[u];
            sk = reinterpret_cast<const float*>(&sc.best_s[par][r][0])[u];
          }, zmax, NU, lane);
          lp = (i0 < 0 || i0 >= p.V1 || !(v0 > -INFINITY)) ? __int_as_float(0x7fffffff) : -(logf(ts) - (z0 - zmax));
        } else if constexpr (SCORED) {   // l of this row: NaN where the label is 0 by the non-finite rule
          const float ts = fold16([&](int r, float& v, float& sk) {
            v = reinterpret_cast<const float*>(&s.best_v[par][r][0])[u];
            sk = reinterpret_cast<const float*>(&sc.best_s[par][r][0])[u];
          }, v0, NU, lane);
          lp = (i0 < 0 || i0 >= p.V1 || !(v0 > -INFINITY)) ? __int_as_float(0x7fffffff) : -logf(ts);
        }
        // lane u < NU decides for utterance u (gigaam/decoding.py:176-205)
        bool act_new = false, run_new = false, moved = false, emitted = false;
        if (lane < NU) {
          int t = s.ctl.t[u];
          const int Lu = s.ctl.L[u];
          int need = s.ctl.need[u];
          if (t < Lu) {
            if constexpr (SCORED) { sc.path[u] += static_cast<double>(lp); sc.rows[u] += 1; }
            if constexpr (SCORED) { r_facc += static_cast<double>(lp); r_frows += 1; }
            if (lab == p.blank) {
              t += 1;
              s.ctl.nsym[u] = 0;
              need = 0;
              moved = true;
            } else {
              const int cnt = s.ctl.cnt[u];
              if (rank == 0 && cnt < p.io.max_out) {
                const size_t o = static_cast<size_t>(group * p.nu + u) * p.io.max_out + cnt;
                p.io.ids[o] = lab;
                p.io.frames[o] = r_fb + t;
                if constexpr (SCORED) p.io.token_logp[o] = lp;
              }
              s.ctl.cnt[u] = cnt + 1;
              s.ctl.label[u] = lab;
              need = 1;   // the state that produced this token becomes the input of the next LSTM step
              emitted = true;
              int ns = s.ctl.nsym[u] + 1;
              if (ns >= p.max_symbols) { t += 1; ns = 0; moved = true; }
              s.ctl.nsym[u] = ns;
            }
            s.ctl.t[u] = t;
            s.ctl.need[u] = need;
            if constexpr (SCORED) {   // a frame is complete when the decoder leaves it
              if (moved) {
                if (rank == 0 && p.io.frame_logp) {
                  const int64_t o = static_cast<int64_t>(group * p.nu + u) * p.io.frame_pitch + r_fb + t - 1;
                  p.io.frame_logp[o] = r_facc;
                  p.io.frame_rows[o] = r_frows;
                }
                r_facc = 0.0;
                r_frows = 0;
              }
            }
          }
          act_new = t < Lu;
          run_new = act_new && need != 0;
        }
        const unsigned am = __ballot_sync(0xffffffffu, act_new), rm = __ballot_sync(0xffffffffu, run_new);
        const unsigned mm = __ballot_sync(0xffffffffu, moved), em = __ballot_sync(0xffffffffu, emitted);
        if (lane == 0) {
          s.ctl.act_m = static_cast<int>(am); s.ctl.run_m = static_cast<int>(rm);
          s.ctl.moved_m = static_cast<int>(mm); s.ctl.emit_m = static_cast<int>(em);
        }
        DBG_T(11);
      }
      ++n_b;
      __syncthreads();
      // what the next rounds need from global memory, requested now and consumed a phase (or a frame) later
      const int moved_m = s.ctl.moved_m, emit_m = s.ctl.emit_m;
      if (tid < kH && moved_m != 0) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            const int u = 4 * hh + cc;
            if ((moved_m >> u) & 1) {
              set_comp(ep[hh], cc, comp(epn[hh], cc));
              const int t1 = s.ctl.t[u] + 1;
              if (t1 < s.ctl.L[u]) set_comp(epn[hh], cc, __ldg(ep_base + (static_cast<size_t>(u) * p.T + t1) * kH));
            }
          }
        }
      }
      if (gate_thread && emit_m != 0) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
          const int u = 4 * hh + lq;
          if ((emit_m >> u) & 1) eg[hh] = __ldg(p.emb_gates + static_cast<size_t>(s.ctl.label[u]) * G + eg_off);
        }
      }
      if constexpr (BOOST) {   // the next joint reads the new slices after the __syncthreads that follows the hid4 build
        if (warp >= kStage0 && emit_m != 0) {
          if (warp == kStage0 && lane < NU && ((emit_m >> lane) & 1)) {
            const int q = __ldg(p.boost.next + static_cast<size_t>(s_q[lane]) * p.V1 + s.ctl.label[lane]);
            s_q[lane] = q >= 0 && q < p.boost.n_states ? q : 0;
          }
          ptx::named_bar_sync<kStageThreads>(1);
          stage(static_cast<unsigned>(emit_m));
        }
      }
      DBG_T(12);
    }
    // ---- end of the group: a fresh call writes the outputs of every row, a resume call those of the streams it advanced and
    // their records
    if (rank == 0 && warp == 0 && lane < NU) {
      const int ug = group * p.nu + lane;
      if (p.io.state ? ((act0 >> lane) & 1) != 0 : (lane < p.nu && ug < p.B)) {
        p.io.counts[ug] = min(s.ctl.cnt[lane], p.io.max_out);
        if constexpr (SCORED) { p.io.path_logp[ug] = static_cast<float>(sc.path[lane]); p.io.path_rows[ug] = sc.rows[lane]; }
        if (DecodeState* st = state_of(p, ug)) {
          st->label = s.ctl.label[lane];
          st->pending = s.ctl.need[lane];
          st->count += s.ctl.cnt[lane] - r_cnt0;
          if constexpr (SCORED) { st->path = sc.path[lane]; st->rows = sc.rows[lane]; }
        }
      }
    }
    if constexpr (BOOST) {   // warp kStage0 is the last writer of q
      if (p.io.state && rank == 0 && warp == kStage0 && lane < NU && ((act0 >> lane) & 1)) state_of(p, group * p.nu + lane)->boost_state = s_q[lane];
    }
    if (p.io.state && tid < NU * kHS) {   // every CTA stores its own units of h, c and pg
      const int u = tid / kHS, j = tid % kHS, k = rank * kHS + j;
      if ((act0 >> u) & 1) {
        DecodeState* st = state_of(p, group * p.nu + u);
        st->h[k] = comp(s.h4[gb][u >> 2][k], u & 3);
        st->c[k] = s.c[gb][u][j];
        st->pg[k] = comp(s.pg4[u >> 2][k], u & 3);
      }
    }
    __syncthreads();   // ctl is re-initialised by warp 0 at the top of the next group
  }
  cluster.sync();      // no CTA may exit while a peer can still store into its shared memory
#ifdef GAM_RNNT_DBG
  if (dbg_on)
    for (int i = 0; i < 16; ++i) g_rnnt_dbg[i] = dbg_acc[i];
#endif
}

struct LaunchState {
  int max_clusters = -1;
  int smem_set = 0;
};

template <int NH, bool GLOB, bool SCORED, bool BOOST>
int launch_nh(RnntClParams& p, int B, int V1, int smem_cap, int* plan, cudaStream_t s) {
  static LaunchState per_device[64];   // function attributes and cluster occupancy are per device
  int dev_index = 0;
  cudaGetDevice(&dev_index);
  LaunchState& st = per_device[dev_index & 63];
  const int cls_per = (V1 + kCl - 1) / kCl;
  const int cls_pad = (cls_per + 3) & ~3;
  const int fixed = smem_before_rows<NH, SCORED, BOOST>(cls_pad);
  int rows_smem = (smem_cap - fixed) / (kWoPitch * 4);
  if (rows_smem < 0) return 1;
  if (rows_smem > cls_per) rows_smem = cls_per;
  if (!GLOB && rows_smem < cls_per) return 1;   // caller picked the wrong variant
  const int smem = fixed + rows_smem * kWoPitch * 4;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCl;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (st.max_clusters < 0 || smem > st.smem_set) {
    if (cudaFuncSetAttribute(rnnt_cluster_kernel<NH, GLOB, SCORED, BOOST>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(rnnt_cluster_kernel<NH, GLOB, SCORED, BOOST>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      cudaGetLastError();
      st.max_clusters = 0;
    } else {
      st.smem_set = smem;
      cfg.gridDim = dim3(kCl);
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, rnnt_cluster_kernel<NH, GLOB, SCORED, BOOST>, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
      st.max_clusters = n;
    }
  }
  if (st.max_clusters <= 0) return 1;
  // spread utterances over as many clusters as can be resident: fewer lock-stepped utterances per cluster
  int nu = (B + st.max_clusters - 1) / st.max_clusters;
  if (nu > 4 * NH) nu = 4 * NH;
  p.nu = nu;
  p.num_groups = (B + nu - 1) / nu;
  p.rows_smem = rows_smem;
  p.cls_pad = cls_pad;
  const int nclusters = p.num_groups < st.max_clusters ? p.num_groups : st.max_clusters;
  cfg.gridDim = dim3(nclusters * kCl);
  if (plan) {
    const int v[7] = {NH, GLOB ? 1 : 0, rows_smem, cls_per, nu, p.num_groups, nclusters};
    for (int i = 0; i < 7; ++i) plan[i] = v[i];
  }
  if (cudaLaunchKernelEx(&cfg, rnnt_cluster_kernel<NH, GLOB, SCORED, BOOST>, p) != cudaSuccess) return -2;
  return 0;
}

}  // namespace

#ifdef GAM_RNNT_DBG
extern "C" int gam_rnnt_debug_read(long long* out16) {
  return cudaMemcpyFromSymbol(out16, g_rnnt_dbg, sizeof(long long) * 16) == cudaSuccess ? 0 : -1;
}
#endif

// returns 0 on success, 1 if the shape is unsupported (pred_hidden != 320) or a 16-CTA cluster cannot be scheduled on
// this device, negative on a launch error.  plan (host, 7 ints, or NULL) receives the launch that was chosen:
// NH, GLOB, class rows per CTA in shared memory, classes per CTA, utterances per group, groups, clusters launched.
// groups of up to 4 utterances (NH = 1) or 8, and whether some class rows have to stay in L2 (GLOB)
template <bool SCORED, bool BOOST>
int launch_sb(RnntClParams& p, bool small, int B, int V1, int cap, int* plan, cudaStream_t s) {
  const int cls_per = (V1 + kCl - 1) / kCl, cls_pad = (cls_per + 3) & ~3;
  if (small) {
    const bool glob = (cap - smem_before_rows<1, SCORED, BOOST>(cls_pad)) / (kWoPitch * 4) < cls_per;
    return glob ? launch_nh<1, true, SCORED, BOOST>(p, B, V1, cap, plan, s) : launch_nh<1, false, SCORED, BOOST>(p, B, V1, cap, plan, s);
  }
  const bool glob = (cap - smem_before_rows<2, SCORED, BOOST>(cls_pad)) / (kWoPitch * 4) < cls_per;
  return glob ? launch_nh<2, true, SCORED, BOOST>(p, B, V1, cap, plan, s) : launch_nh<2, false, SCORED, BOOST>(p, B, V1, cap, plan, s);
}

// io.token_logp (or NULL: the unscored kernel) selects the scored instantiation, boost (or NULL) the boosted one.
int launch_rnnt_greedy(const float* encproj, const float* emb_gates, const float* whhT, const float* wpT, const float* bp,
                       const float* wo, const float* bo, int B, int T, int H, int V1, int blank, int max_symbols, const GreedyIo& io,
                       const BoostGraph* boost, int* plan, cudaStream_t s) {
  if (H != kH) return 1;
  struct DeviceLimits {
    int smem_cap = 0, clusters_hint = 0;
  };
  static DeviceLimits per_device[64];
  int dev = 0;
  cudaGetDevice(&dev);
  DeviceLimits& lim = per_device[dev & 63];
  if (lim.smem_cap == 0) {
    cudaDeviceGetAttribute(&lim.smem_cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // GPCs rarely hold more than one 16-CTA cluster each (a 132-SM H100 has 7 or 8 GPCs)
    lim.clusters_hint = sms / kCl - 2 < 1 ? 1 : sms / kCl - 2;
  }
  const bool scored = io.token_logp != nullptr;
  if (scored && (!io.path_logp || !io.path_rows)) return -1;
  RnntClParams p;
  p.encproj = encproj; p.emb_gates = emb_gates; p.whhT = whhT; p.wpT = wpT; p.bp = bp; p.wo = wo; p.bo = bo;
  p.B = B; p.T = T; p.V1 = V1; p.blank = blank; p.max_symbols = max_symbols;
  p.io = io;
  p.boost = boost ? *boost : BoostGraph{};
  // groups of up to 4 utterances while every group still gets its own cluster, else groups of up to 8
  const bool small = B <= 4 * lim.clusters_hint;
  const int cap = lim.smem_cap;
  if (boost) return scored ? launch_sb<true, true>(p, small, B, V1, cap, plan, s) : launch_sb<false, true>(p, small, B, V1, cap, plan, s);
  return scored ? launch_sb<true, false>(p, small, B, V1, cap, plan, s) : launch_sb<false, false>(p, small, B, V1, cap, plan, s);
}

}  // namespace gam
