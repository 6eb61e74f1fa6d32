// C-ABI + host engine of libgigaam_b200.so: weight/plan bookkeeping, TMA descriptor construction,
// and the kernel sequence of the path.  No compute lives here and nothing here falls back to a CPU
// or library implementation: every stage is one of the hand-written kernels in this directory.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/gigaam_b200.h"
#include "comm.h"
#include "gemm_params.cuh"
#include "kernels.h"
#include "launch.cuh"

namespace gam {

// ------------------------------------------------------------------ driver entry point for TMA descriptors
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int init_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || fn == nullptr ||
      q != cudaDriverEntryPointSuccess)
    return -1;
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return 0;
}

// 2-D row-major tensor [rows, cols] of `esz`-byte elements with row pitch ld_elems; box = [box_rows, box_cols], SWIZZLE_128B
static int make_tmap_2d(CUtensorMap* m, CUtensorMapDataType type, uint64_t esz, const void* base, uint64_t rows, uint64_t cols,
                        uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols) {
  if (init_encode() != 0) return -1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * esz};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, type, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}
int make_tmap_2d_f16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                     uint32_t box_cols) {
  return make_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, rows, cols, ld_elems, box_rows, box_cols);
}
static int make_tmap_2d_f32(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                            uint32_t box_cols) {
  return make_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, rows, cols, ld_elems, box_rows, box_cols);
}

// GEMM output columns [rows, cols] at `base`, pitch ld_elems, in boxes of one store slot of the GEMM
// (64 rows x 128 bytes: 64 fp16 or 32 fp32 columns).  Nonzero when TMA cannot address it (base or pitch not 16-byte
// aligned): the launch then stores every tile directly.
static int make_tmap_out(CUtensorMap* m, const void* base, bool f32, uint64_t rows, uint64_t cols, uint64_t ld_elems) {
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0 || (ld_elems * (f32 ? 4 : 2)) % 16 != 0) return -1;
  return f32 ? make_tmap_2d_f32(m, base, rows, cols, ld_elems, 64, 32) : make_tmap_2d_f16(m, base, rows, cols, ld_elems, 64, 64);
}

// 4-D channels-last activation [B, T1, F1, C] fp16 for the stride-2 3x3 conv: box = 8 time x 16 freq x 64 ch,
// traversal stride 2 on time and freq (so boxDim is 16 / 32 elements in tensor coordinates).
static int make_tmap_conv4d(CUtensorMap* m, const void* base, uint64_t B, uint64_t T1, uint64_t F1, uint64_t C) {
  if (init_encode() != 0) return -1;
  cuuint64_t dims[4] = {C, F1, T1, B};
  cuuint64_t strides[3] = {C * 2, F1 * C * 2, T1 * F1 * C * 2};
  cuuint32_t box[4] = {64, 32, 16, 1};
  cuuint32_t estr[4] = {1, 2, 2, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

// 3-D time-major activation [B, T, C] fp16 for the stride-2 conv1d: box = 128 output frames (256 input frames
// traversed with stride 2) x 64 channels
static int make_tmap_conv3d(CUtensorMap* m, const void* base, uint64_t B, uint64_t T, uint64_t C) {
  if (init_encode() != 0) return -1;
  cuuint64_t dims[3] = {C, T, B};
  cuuint64_t strides[2] = {C * 2, T * C * 2};
  cuuint32_t box[3] = {64, 256, 1};
  cuuint32_t estr[3] = {1, 2, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

struct LayerMaps {
  CUtensorMap ff1_w1, ff1_w2, w_qk, w_v, w_o, pw1, pw2, ff2_w1, ff2_w2;
  CUtensorMap w_qkv_rel, pos_proj;   // rel_pos attention only
  CUtensorMap w_qkv;                 // rotary: [W_q ; W_k ; W_v] when the caller packed them contiguously
  bool qkv_merged = false;
};

struct Plan {
  int B = 0;
  int64_t M = 0;
  void* ws = nullptr;
  // geometry
  int T1 = 0, F1 = 0, T2 = 0, F2 = 0, R = 0;
  // workspace carve-up
  int *len0 = nullptr, *len1 = nullptr, *len2 = nullptr;
  // packed-row plan (pack_plan_kernel): frames kept per utterance, their prefix sum [B + 1], the live row count, the
  // stage-1 frames that are produced, and row -> (utterance, frame)
  int *plen = nullptr, *cu = nullptr, *rows_dev = nullptr, *run1 = nullptr, *row_b = nullptr, *row_t = nullptr;
  __half *s1 = nullptr, *s2 = nullptr, *a16 = nullptr, *r16 = nullptr, *big16 = nullptr, *o16 = nullptr, *g16 = nullptr;
  __half* melT = nullptr;   // conv1d subsampling: time-major fp16 copy of the log-mel
  CUtensorMap m_melT, m_s1_3d;
  float* x = nullptr;
  int64_t bytes = 0;
  CUtensorMap m_s1, m_s2, m_a16, m_r16, m_hid, m_qkv, m_qkv4, m_o16;
  // GEMM outputs (make_tmap_out): big16 at d_ff / 3d / 4d columns, its q|k and v column ranges of the unmerged projection, g16,
  // and x (fp32, the sub_out GEMM)
  CUtensorMap o_hid, o_qkv, o_qkv4, o_qk, o_v, o_g16, o_x;
};

}  // namespace gam

using namespace gam;

struct gam_handle {
  gam_config cfg;
  gam_weights w;
  std::vector<gam_layer_weights> layers;
  std::vector<LayerMaps> lmaps;
  CUtensorMap m_sub2_w, m_sub_out_w;
  CUtensorMap m_dft_w, m_lm_a;   // tensor-core front end: split DFT basis / frame matrix (cached per workspace)
  const void* lm_A = nullptr;
  int64_t lm_F = 0;
  int device = 0;
  int gemm_clusters = 0;   // co-resident clusters of the GEMM kernel (gemm_init)
  int max_t = GAM_REL_POS_MAX_T;   // longest T' (cfg.max_encoded_frames, 0 = default); rel_pos tables have 2*max_t-1 rows
  int64_t launches = 0;
  int test_gemm_slots = 0;   // the last gam_test_gemm launch could store through the shared-memory slots
  void* comm = nullptr;      // ncclComm_t of gam_comm_init
  int comm_rank = 0, comm_nranks = 1;
  std::string err;
  std::vector<Plan*> plans;
  // optional per-launch CUDA-event timing (bench.py's roofline leg); never active during graph capture
  bool prof = false;
  std::vector<cudaEvent_t> prof_ev;   // start/stop pairs
  std::vector<int> prof_cls;
};

// kernel classes reported by gam_profile_end
enum ProfClass : int {
  PC_LOGMEL = 0, PC_SUB_CONV1, PC_GEMM_CONV2, PC_GEMM_SUBOUT, PC_GEMM_FFN_UP, PC_GEMM_FFN_DOWN, PC_GEMM_QKV, PC_GEMM_PROJ,
  PC_GEMM_GLU, PC_LAYERNORM, PC_ATTENTION, PC_DWCONV, PC_CTC_ARGMAX, PC_CTC_COLLAPSE, PC_RNNT_ENCPROJ, PC_RNNT_GREEDY,
  PC_MISC, PC_CTC_LOG_PROBS, PC_RNNT_JOINT, PC_RNNT_PREDICT, PC_EMO_HEAD, PC_HEAD_BACKWARD, PC_ALIGN, PC_EMO_FRAME_LOGITS, PC_EMO_SPANS, PC_COUNT
};

struct ProfScope {
  gam_handle* h;
  cudaStream_t s;
  ProfScope(gam_handle* h_, int cls, cudaStream_t s_) : h(h_), s(s_) {
    h->launches += 1;
    if (!h->prof) return;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    h->prof_ev.push_back(a);
    h->prof_ev.push_back(b);
    h->prof_cls.push_back(cls);
    cudaEventRecord(a, s);
  }
  ~ProfScope() {
    if (h->prof) cudaEventRecord(h->prof_ev.back(), s);
  }
};
#define PROF(cls) ProfScope prof_scope__(h, cls, s)

namespace {

int fail(gam_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  return code;
}

// A workspace carved into 1 KiB-aligned pieces; base == nullptr only sizes it.  `off` is the size with every piece rounded
// up, `end` where the last piece ends.
struct Carve {
  uint8_t* base;
  int64_t off = 0, end = 0;
  template <typename T = float>
  T* take(int64_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    end = off + count * static_cast<int64_t>(sizeof(T));
    off = align_up(end, 1024);
    return p;
  }
};

// The caller's workspace for a layout of `need` bytes: its base, rounded up to 1 KiB when `slack` (the layout's size query
// adds 1 KiB for that); nullptr, with the error set, when it is NULL or smaller than need.
uint8_t* workspace_base(gam_handle* h, const char* what, void* workspace, int64_t workspace_bytes, int64_t need, bool slack) {
  if (workspace == nullptr || workspace_bytes < need) {
    fail(h, -1, "%s: workspace too small: need %lld bytes, got %lld", what, (long long)need, (long long)workspace_bytes);
    return nullptr;
  }
  const uintptr_t p = reinterpret_cast<uintptr_t>(workspace);
  return reinterpret_cast<uint8_t*>(slack ? (p + 1023) & ~uintptr_t(1023) : p);
}

int sub_out_len(int len, int k, int pad) {
  // floor((len + 2p - k) / 2 + 1) with float semantics of the reference (encoder.py:86-90)
  float l = static_cast<float>(len);
  l = floorf((l + (2 * pad - k)) / 2.0f + 1.0f);
  return static_cast<int>(l);
}

void plan_geometry(const gam_handle* h, int B, int64_t M, Plan* p) {
  const gam_config& c = h->cfg;
  const int k = c.subs_kernel_size, pad = (k - 1) / 2;
  p->B = B;
  p->M = M;
  p->T1 = sub_out_len(static_cast<int>(M), k, pad);
  p->T2 = sub_out_len(p->T1, k, pad);
  p->F1 = c.subsampling == 0 ? sub_out_len(c.feat_in, k, pad) : 1;
  p->F2 = c.subsampling == 0 ? sub_out_len(p->F1, k, pad) : 1;
  p->R = B * p->T2;
}

// carve the workspace; returns total bytes.  base may be null (size query).
int64_t plan_carve(const gam_handle* h, Plan* p, uint8_t* base) {
  const gam_config& c = h->cfg;
  const int64_t d = c.d_model, R = p->R, B = p->B;
  const int64_t nqkv = (c.self_attention == 1 ? 4 : 3) * d;   // rel_pos carries q twice (q+u, q+v)
  const int64_t wide = (c.d_ff > nqkv ? c.d_ff : nqkv);
  int64_t off = 0;
  auto take = [&](int64_t bytes) -> uint8_t* {
    uint8_t* ptr = base ? base + off : nullptr;
    off += align_up(bytes, 1024);
    return ptr;
  };
  p->len0 = reinterpret_cast<int*>(take(B * 4));
  p->len1 = reinterpret_cast<int*>(take(B * 4));
  p->len2 = reinterpret_cast<int*>(take(B * 4));
  p->plen = reinterpret_cast<int*>(take(B * 4));
  p->run1 = reinterpret_cast<int*>(take(B * 4));
  p->cu = reinterpret_cast<int*>(take((B + 1) * 4));
  p->rows_dev = reinterpret_cast<int*>(take(4));
  p->row_b = reinterpret_cast<int*>(take(R * 4));
  p->row_t = reinterpret_cast<int*>(take(R * 4));
  p->x = reinterpret_cast<float*>(take(R * d * 4));
  p->a16 = reinterpret_cast<__half*>(take(R * d * 2));
  p->r16 = reinterpret_cast<__half*>(take(R * d * 2));
  p->big16 = reinterpret_cast<__half*>(take(R * wide * 2));
  p->o16 = reinterpret_cast<__half*>(take(R * d * 2));
  p->g16 = reinterpret_cast<__half*>(take(R * d * 2));
  p->s2 = reinterpret_cast<__half*>(take(R * static_cast<int64_t>(p->F2) * d * 2));
  p->s1 = reinterpret_cast<__half*>(take(B * static_cast<int64_t>(p->T1) * p->F1 * d * 2));
  p->melT = reinterpret_cast<__half*>(take(c.subsampling == 1 ? B * p->M * static_cast<int64_t>(c.feat_in) * 2 : 0));
  return off;
}

int64_t decode_ws_bytes(const gam_handle* h, int B, int T) {
  // CTC: labels [B*T] i32 ; RNNT: encproj [B*T, joint_hidden] f32
  const int64_t R = static_cast<int64_t>(B) * T;
  int64_t a = align_up(R * 4, 1024);
  int64_t b = align_up(R * (h->cfg.joint_hidden > 0 ? h->cfg.joint_hidden : 1) * 4, 1024);
  return a + b;
}

Plan* get_plan(gam_handle* h, int B, int64_t M, void* ws, int64_t ws_bytes) {
  for (Plan* p : h->plans)
    if (p->B == B && p->M == M && p->ws == ws) return p;
  Plan* p = new Plan();
  plan_geometry(h, B, M, p);
  p->ws = ws;
  p->bytes = plan_carve(h, p, static_cast<uint8_t*>(ws));
  if (p->bytes > ws_bytes) {
    fail(h, -1, "workspace too small: need %lld bytes, got %lld", (long long)p->bytes, (long long)ws_bytes);
    delete p;
    return nullptr;
  }
  const gam_config& c = h->cfg;
  const uint64_t d = c.d_model, R = p->R;
  int rc = 0;
  if (c.subsampling == 0) {
    rc |= make_tmap_conv4d(&p->m_s1, p->s1, B, p->T1, p->F1, d);
    rc |= make_tmap_2d_f16(&p->m_s2, p->s2, R, static_cast<uint64_t>(p->F2) * d, static_cast<uint64_t>(p->F2) * d, 128, 64);
  } else {
    rc |= make_tmap_conv3d(&p->m_melT, p->melT, B, static_cast<uint64_t>(p->M), c.feat_in);
    rc |= make_tmap_conv3d(&p->m_s1_3d, p->s1, B, p->T1, d);
  }
  rc |= make_tmap_2d_f16(&p->m_a16, p->a16, R, d, d, 128, 64);
  rc |= make_tmap_2d_f16(&p->m_r16, p->r16, R, d, d, 128, 64);
  rc |= make_tmap_2d_f16(&p->m_hid, p->big16, R, c.d_ff, c.d_ff, 128, 64);
  rc |= make_tmap_2d_f16(&p->m_qkv, p->big16, R, 3 * d, 3 * d, 128, 64);
  rc |= make_tmap_2d_f16(&p->m_qkv4, p->big16, R, 4 * d, 4 * d, 128, 64);
  rc |= make_tmap_2d_f16(&p->m_o16, p->o16, R, d, d, 128, 64);
  rc |= make_tmap_out(&p->o_hid, p->big16, false, R, c.d_ff, c.d_ff);
  rc |= make_tmap_out(&p->o_qkv, p->big16, false, R, 3 * d, 3 * d);
  rc |= make_tmap_out(&p->o_qkv4, p->big16, false, R, 4 * d, 4 * d);
  rc |= make_tmap_out(&p->o_qk, p->big16, false, R, 2 * d, 3 * d);
  rc |= make_tmap_out(&p->o_v, p->big16 + 2 * d, false, R, d, 3 * d);
  rc |= make_tmap_out(&p->o_g16, p->g16, false, R, d, d);
  rc |= make_tmap_out(&p->o_x, p->x, true, R, d, d);
  if (rc != 0) {
    fail(h, -2, "cuTensorMapEncodeTiled failed for activation maps (rc=%d)", rc);
    delete p;
    return nullptr;
  }
  if (h->plans.size() >= 16) {
    delete h->plans.front();
    h->plans.erase(h->plans.begin());
  }
  h->plans.push_back(p);
  return p;
}

// gam_test_gemm's kind for the DFT power epilogue (launch_gemm_power); kinds 0-4 are GemmKind
constexpr int kTestGemmPower = 7;

// Unit-test entry points only: copies n device ints to the host (synchronising the stream) so that a hook can refuse row
// maps that would send its kernel outside the caller's buffers.  Returns 0 on success.
int dev_ints(const int32_t* p, int n, std::vector<int>& v, cudaStream_t s) {
  v.assign(n > 0 ? n : 0, 0);
  if (n <= 0) return 0;
  if (cudaMemcpyAsync(v.data(), p, static_cast<size_t>(n) * sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) return -1;
  return cudaStreamSynchronize(s) == cudaSuccess ? 0 : -1;
}

#define GAM_CHECK_LAUNCH(h, what)                                                           \
  do {                                                                                        \
    cudaError_t e__ = cudaGetLastError(); /* reads AND clears: one failed launch must not poison later calls */ \
    if (e__ != cudaSuccess) return fail(h, -3, "%s: %s", what, cudaGetErrorString(e__));      \
  } while (0)

}  // namespace

extern "C" {

int gam_version(void) { return 100; }

const char* gam_last_error(const gam_handle* h) { return h ? h->err.c_str() : "null handle"; }

int64_t gam_launch_count(const gam_handle* h) { return h ? h->launches : 0; }

int gam_create(const gam_config* cfg, const gam_weights* w, int device, gam_handle** out) {
  if (!cfg || !w || !out) return -1;
  *out = nullptr;
  gam_handle* h = new gam_handle();
  h->cfg = *cfg;
  h->w = *w;
  h->device = device;
  *out = h;  // returned even on failure so the caller can read gam_last_error()
  const gam_config& c = h->cfg;
  if (c.subsampling != 0 && c.subsampling != 1) return fail(h, -10, "unknown subsampling type %d", c.subsampling);
  if (c.subsampling == 1 && (c.feat_in % 64 != 0 || (c.subs_kernel_size & 1) == 0))
    return fail(h, -10, "conv1d subsampling needs feat_in %% 64 == 0 and an odd kernel size");
  if (c.self_attention != 0 && c.self_attention != 1) return fail(h, -10, "unknown self_attention type %d", c.self_attention);
  if (c.d_model != 768 || c.n_heads <= 0 || c.d_model % c.n_heads != 0 || (c.d_model / c.n_heads) % 16 != 0)
    return fail(h, -10, "unsupported d_model/n_heads (%d/%d): kernels are specialised for d_model 768, d_k %% 16 == 0",
                c.d_model, c.n_heads);
  {  // refused here, not at the first encode: the attention launchers check the same limits
    const int dk = c.d_model / c.n_heads, dk_max = c.self_attention == 0 ? GAM_ROTARY_MAX_DK : GAM_REL_POS_MAX_DK;
    if (dk > dk_max)
      return fail(h, -10, "%s attention runs heads of d_k <= %d, but d_model %d / n_heads %d gives d_k = %d",
                  c.self_attention == 0 ? "rotary" : "rel_pos", dk_max, c.d_model, c.n_heads, dk);
  }
  if (c.d_ff % 256 != 0 || (c.subsampling == 0 && c.subs_kernel_size != 3)) return fail(h, -10, "unsupported d_ff / subs_kernel_size");
  if (c.win_length != c.n_fft) return fail(h, -10, "win_length != n_fft is not supported");
  if (c.n_mels < 1 || c.n_mels > 64) return fail(h, -10, "n_mels %d outside [1, 64]: the log-mel kernels hold 64 mel rows", c.n_mels);
  if (c.max_encoded_frames != 0) {
    if (c.max_encoded_frames < GAM_REL_POS_MAX_T || c.max_encoded_frames > c.pos_emb_max_len)
      return fail(h, -10, "max_encoded_frames %d outside [%d, pos_emb_max_len = %d]: the rotary and relative-position tables "
                  "have pos_emb_max_len rows", c.max_encoded_frames, GAM_REL_POS_MAX_T, c.pos_emb_max_len);
    h->max_t = c.max_encoded_frames;
  }
  if (c.head == 3) {
    if (c.num_classes < 1 || c.num_classes > kPoolMaxClasses)
      return fail(h, -10, "emo head: %d classes outside [1, %d]", c.num_classes, kPoolMaxClasses);
    if (!w->emo_w || !w->emo_b) return fail(h, -10, "emo head: emo_w / emo_b missing");
  }
  if (cudaSetDevice(device) != cudaSuccess) return fail(h, -11, "cudaSetDevice(%d) failed", device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(h, -11, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)
    return fail(h, -12, "sm_90a kernels need a Hopper (cc 9.0) device, found cc %d.%d", prop.major, prop.minor);
  if (init_encode() != 0) return fail(h, -13, "cuTensorMapEncodeTiled entry point not available");
  if (gemm_init(&h->gemm_clusters) != 0) return fail(h, -14, "GEMM kernel set-up (shared memory opt-in, cluster occupancy) failed: %s", cudaGetErrorString(cudaGetLastError()));
  h->layers.assign(w->layers, w->layers + c.n_layers);
  h->w.layers = h->layers.data();
  h->lmaps.resize(c.n_layers);
  const uint64_t d = c.d_model, ff = c.d_ff;
  int rc = 0;
  for (int l = 0; l < c.n_layers; ++l) {
    const gam_layer_weights& lw = h->layers[l];
    LayerMaps& lm = h->lmaps[l];
    rc |= make_tmap_2d_f16(&lm.ff1_w1, lw.ff1_w1, ff, d, d, 128, 64);
    rc |= make_tmap_2d_f16(&lm.ff1_w2, lw.ff1_w2, d, ff, ff, 128, 64);
    if (c.self_attention == 0) {
      rc |= make_tmap_2d_f16(&lm.w_qk, lw.w_qk, 2 * d, d, d, 128, 64);
      rc |= make_tmap_2d_f16(&lm.w_v, lw.w_v, d, d, d, 128, 64);
      // W_v directly behind W_qk (and b_v behind b_qk): q, k and v projections run as one launch (launch_gemm_dual_a)
      lm.qkv_merged = static_cast<const char*>(lw.w_v) == static_cast<const char*>(lw.w_qk) + 2 * d * d * 2 && lw.b_v == lw.b_qk + 2 * d;
      if (lm.qkv_merged) rc |= make_tmap_2d_f16(&lm.w_qkv, lw.w_qk, 3 * d, d, d, 128, 64);
    } else {
      if (!lw.w_qkv_rel || !lw.b_qkv_rel || !lw.pos_proj) return fail(h, -10, "layer %d: rel_pos weights missing", l);
      rc |= make_tmap_2d_f16(&lm.w_qkv_rel, lw.w_qkv_rel, 4 * d, d, d, 128, 64);
      rc |= make_tmap_2d_f16(&lm.pos_proj, lw.pos_proj, 2 * static_cast<uint64_t>(h->max_t) - 1, d, d, 128, 64);
    }
    rc |= make_tmap_2d_f16(&lm.w_o, lw.w_o, d, d, d, 128, 64);
    rc |= make_tmap_2d_f16(&lm.pw1, lw.pw1_w, 2 * d, d, d, 128, 64);
    rc |= make_tmap_2d_f16(&lm.pw2, lw.pw2_w, d, d, d, 128, 64);
    rc |= make_tmap_2d_f16(&lm.ff2_w1, lw.ff2_w1, ff, d, d, 128, 64);
    rc |= make_tmap_2d_f16(&lm.ff2_w2, lw.ff2_w2, d, ff, ff, 128, 64);
  }
  const int pad = (c.subs_kernel_size - 1) / 2;
  const int F1 = sub_out_len(c.feat_in, c.subs_kernel_size, pad), F2 = sub_out_len(F1, c.subs_kernel_size, pad);
  if (c.subsampling == 0) {
    if (F1 != 32 || F2 != 16) return fail(h, -10, "conv2d subsampling kernels are specialised for feat_in 64 (F1=32,F2=16)");
    rc |= make_tmap_2d_f16(&h->m_sub2_w, w->sub2_w, d, 9 * d, 9 * d, 128, 64);
    rc |= make_tmap_2d_f16(&h->m_sub_out_w, w->sub_out_w, d, static_cast<uint64_t>(F2) * d, static_cast<uint64_t>(F2) * d, 128, 64);
  } else {
    const uint64_t k1 = static_cast<uint64_t>(c.subs_kernel_size) * c.feat_in, k2 = static_cast<uint64_t>(c.subs_kernel_size) * d;
    rc |= make_tmap_2d_f16(&h->m_sub2_w, w->c1d_w1, d, k1, k1, 128, 64);        // stage 1: [d, taps * feat_in]
    rc |= make_tmap_2d_f16(&h->m_sub_out_w, w->c1d_w2, d, k2, k2, 128, 64);     // stage 2: [d, taps * d]
  }
  if (w->dft_w != nullptr) {
    const uint64_t kk = 3 * static_cast<uint64_t>((c.n_fft + 63) / 64 * 64);
    rc |= make_tmap_2d_f16(&h->m_dft_w, w->dft_w, 512, kk, kk, 128, 64);
  }
  if (rc != 0) return fail(h, -2, "cuTensorMapEncodeTiled failed for weight maps (rc=%d)", rc);
  return 0;
}

void gam_destroy(gam_handle* h) {
  if (!h) return;
  for (Plan* p : h->plans) delete p;
  comm_destroy(h->comm);
  delete h;
}

int64_t gam_logmel_frames(const gam_handle* h, int64_t n) {
  const gam_config& c = h->cfg;
  if (c.center) return n / c.hop_length + 1;
  return n < c.win_length ? 0 : (n - c.win_length) / c.hop_length + 1;
}

int64_t gam_encoded_frames(const gam_handle* h, int64_t M) {
  Plan p;
  plan_geometry(h, 1, M, &p);
  return p.T2;
}

int64_t gam_decode_workspace_bytes(const gam_handle* h, int32_t B, int32_t T) { return decode_ws_bytes(h, B, T) + 1024; }

// the scored decoders also keep the CTC per-frame l [B*T] f32 after the labels
static int64_t scored_extra_bytes(int32_t B, int32_t T) { return align_up(static_cast<int64_t>(B) * T * 4, 1024); }
int64_t gam_decode_scored_workspace_bytes(const gam_handle* h, int32_t B, int32_t T) {
  return decode_ws_bytes(h, B, T) + scored_extra_bytes(B, T) + 1024;
}

int64_t gam_workspace_bytes(const gam_handle* h, int32_t B, int64_t M) {
  Plan p;
  plan_geometry(h, B, M, &p);
  return plan_carve(h, &p, nullptr) + decode_ws_bytes(h, B, p.T2) + 4096;
}

int gam_logmel(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, float* mel, void* stream) {
  const gam_config& c = h->cfg;
  const int64_t M = gam_logmel_frames(h, n_samples);
  if (M <= 0) return fail(h, -1, "waveform too short: %lld samples", (long long)n_samples);
  if (c.center && n_samples <= c.n_fft / 2) return fail(h, -1, "reflect padding needs more than n_fft/2 samples");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    PROF(PC_LOGMEL);
    if (launch_logmel(wav, B, static_cast<int>(n_samples), static_cast<int>(M), h->w.window, h->w.dft_cos, h->w.dft_sin,
                      h->w.mel_fb, mel, c.n_fft, c.hop_length, c.center, c.n_mels, s) != 0)
      return fail(h, -1, "logmel: unsupported n_fft/n_mels (%d/%d)", c.n_fft, c.n_mels);
  }
  GAM_CHECK_LAUNCH(h, "logmel");
  return 0;
}

static inline int logmel_kp(const gam_config& c) { return (c.n_fft + 63) / 64 * 64; }

// workspace of gam_logmel_tc: A' f16 [F, 3 Kp] | power f32 [F, 256] | per-frame exponent i32 [F] (frames_split_kernel)
int64_t gam_logmel_workspace_bytes(const gam_handle* h, int32_t B, int64_t n_samples) {
  const int64_t F = static_cast<int64_t>(B) * gam_logmel_frames(h, n_samples);
  return align_up(F * 3 * logmel_kp(h->cfg) * 2, 1024) + align_up(F * 256 * 4, 1024) + align_up(F * 4, 1024) + 2048;
}

int gam_logmel_tc(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, float* mel, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  const gam_config& c = h->cfg;
  if (!h->w.dft_w || !h->w.mel_lo || !h->w.mel_hi) return fail(h, -1, "logmel_tc: split DFT basis not provided");
  if (c.n_fft / 2 + 1 > 256) return fail(h, -1, "logmel_tc: n_fft %d exceeds 256 bins", c.n_fft);
  const int64_t M = gam_logmel_frames(h, n_samples);
  if (M <= 0) return fail(h, -1, "waveform too short: %lld samples", (long long)n_samples);
  if (c.center && n_samples <= c.n_fft / 2) return fail(h, -1, "reflect padding needs more than n_fft/2 samples");
  if (workspace_bytes < gam_logmel_workspace_bytes(h, B, n_samples)) return fail(h, -1, "logmel_tc: workspace too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int Kp = logmel_kp(c);
  const int64_t F = static_cast<int64_t>(B) * M;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  ws = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
  __half* A = reinterpret_cast<__half*>(ws);
  float* P = reinterpret_cast<float*>(ws + align_up(F * 3 * Kp * 2, 1024));
  int* fexp = reinterpret_cast<int*>(ws + align_up(F * 3 * Kp * 2, 1024) + align_up(F * 256 * 4, 1024));
  if (h->lm_A != A || h->lm_F != F) {
    if (make_tmap_2d_f16(&h->m_lm_a, A, F, 3 * Kp, 3 * Kp, 128, 64) != 0) return fail(h, -2, "logmel_tc: tensor map encode failed");
    h->lm_A = A;
    h->lm_F = F;
  }
  {
    PROF(PC_LOGMEL);
    if (launch_frames_split(wav, B, static_cast<int>(n_samples), static_cast<int>(M), h->w.window, A, fexp, c.n_fft, Kp, c.hop_length,
                            c.center, s) != 0)
      return fail(h, -4, "logmel_tc: frame split launch rejected (n_fft %d)", c.n_fft);
  }
  {
    PROF(PC_LOGMEL);
    if (launch_gemm_power(&h->m_lm_a, &h->m_dft_w, static_cast<int>(F), 512, 3 * Kp, P, 256, h->gemm_clusters, s) != 0)
      return fail(h, -4, "logmel_tc: DFT GEMM launch rejected");
  }
  {
    PROF(PC_LOGMEL);
    if (launch_mel_log(P, fexp, 256, B, static_cast<int>(M), c.n_fft / 2 + 1, h->w.mel_fb, h->w.mel_lo, h->w.mel_hi, mel, c.n_mels,
                       s) != 0)
      return fail(h, -4, "logmel_tc: mel projection launch rejected (n_mels %d)", c.n_mels);
  }
  GAM_CHECK_LAUNCH(h, "logmel_tc");
  return 0;
}

int gam_encode(gam_handle* h, const float* mel, const int64_t* mel_len, int32_t B, int64_t M, void* workspace,
               int64_t workspace_bytes, float* enc, int32_t* enc_len, int32_t n_layers_run, void* stream) {
  const gam_config& c = h->cfg;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (B <= 0 || M <= 0) return fail(h, -1, "encode: empty batch (B=%d, M=%lld); callers skip the call for an empty shard", B, (long long)M);
  Plan* p = get_plan(h, B, M, workspace, workspace_bytes);
  if (!p) return -1;
  if (p->T2 <= 0) return fail(h, -1, "input too short for the subsampling (M=%lld)", (long long)M);
  if (p->T2 > h->max_t)
    return fail(h, -1, "T'=%d exceeds the attention kernels' %d-frame limit (%.1f s of audio); cut the recording into segments "
                "(transcribe_longform does)", p->T2, h->max_t, h->max_t * 0.04);
  const int d = c.d_model, R = p->R, ncl = h->gemm_clusters;
  const int L = (n_layers_run < 0 || n_layers_run > c.n_layers) ? c.n_layers : n_layers_run;
  int rc = 0;

  // Varlen execution: from the second subsampling stage on, the path keeps only the frames that exist.  Utterance b owns rows
  // cu[b] .. cu[b] + plen[b] of every activation matrix (plen = its subsampled length; a batch of one keeps all T' frames,
  // like the reference's mask-free single-utterance attention); the live row count stays on the device (rows_dev), so the
  // same launch sequence -- and a captured CUDA graph of it -- serves every mix of lengths.  Grids are sized for R = B*T'.
  {
    PROF(PC_MISC);
    launch_pack_plan(reinterpret_cast<const long long*>(mel_len), B, 2 * ((c.subs_kernel_size - 1) / 2) - c.subs_kernel_size,
                     static_cast<int>(M), p->T1, p->T2, p->len0, p->len1, p->len2, p->plen, p->run1, p->cu, p->rows_dev, p->row_b,
                     p->row_t, s);
  }
  const int* rdev = p->rows_dev;
  if (c.subsampling == 0) {
    {
      PROF(PC_SUB_CONV1);
      rc |= launch_subsample_conv1(mel, p->len0, p->len1, p->run1, h->w.sub1_w, h->w.sub1_b, p->s1, B, static_cast<int>(M), c.feat_in,
                                   p->T1, p->F1, d, s);
    }
    {
      PROF(PC_GEMM_CONV2);
      rc |= launch_gemm_conv(&p->m_s1, &h->m_sub2_w, B, p->T2, d, d, h->w.sub2_b, p->len2, p->cu, p->plen, p->s2, d, ncl, s);
    }
    GAM_CHECK_LAUNCH(h, "subsampling");
    if (rc) return fail(h, -4, "subsampling launch rejected (rc=%d)", rc);
    {
      PROF(PC_GEMM_SUBOUT);
      rc |= launch_gemm(GEMM_BIAS_F32, &p->m_s2, &h->m_sub_out_w, R, d, p->F2 * d, h->w.sub_out_b, nullptr, p->x, d, 1.f, ncl, s, 0, rdev,
                        &p->o_x);
    }
  } else {
    // conv1d subsampling (gigaam/encoder.py:59-70 with Conv1d): two k-tap / stride-2 implicit GEMMs over time-major data
    {
      PROF(PC_SUB_CONV1);
      launch_mel_to_tmajor_f16(mel, p->len0, p->melT, B, c.feat_in, static_cast<int>(M), s);
    }
    {
      PROF(PC_GEMM_CONV2);
      rc |= launch_gemm_conv1d(&p->m_melT, &h->m_sub2_w, B, p->T1, c.feat_in, c.subs_kernel_size, d, h->w.c1d_b1, p->len1, nullptr,
                               nullptr, p->s1, d, 0, ncl, s);   // stage 1 stays [B, T1]: stage 2 fetches it with 3-D TMA boxes
    }
    {
      PROF(PC_GEMM_SUBOUT);
      rc |= launch_gemm_conv1d(&p->m_s1_3d, &h->m_sub_out_w, B, p->T2, d, c.subs_kernel_size, d, h->w.c1d_b2, p->len2, p->cu,
                               p->plen, p->x, d, 1, ncl, s);
    }
    GAM_CHECK_LAUNCH(h, "subsampling");
    if (rc) return fail(h, -4, "conv1d subsampling launch rejected (rc=%d)", rc);
  }
  // Direction plan of a layer (GemmParams::reverse): every kernel walks the rows in the direction OPPOSITE to the one its
  // main input was written in, so that it starts on what is still in L2.  U = ascending, D = descending:
  //   LN_ff1 D | FF1-up U | FF1-down D | LN_att U | QKV D | attention U | proj D | LN_conv U | pw1 D | depthwise U | pw2 D |
  //   LN_ff2 U | FF2-up D | FF2-down U | LN_out (+ next LN_ff1) D
  constexpr int zz = 1;
  if (L == 0) {   // n_layers_run == 0: the caller wants the pre_encode output
    PROF(PC_MISC);
    launch_unpack_rows(p->x, nullptr, nullptr, p->cu, p->plen, enc, B, p->T2, 0, s);
  } else {
    PROF(PC_LAYERNORM);
    launch_ln_f16(p->x, h->layers[0].ln_ff1_g, h->layers[0].ln_ff1_b, p->a16, R, rdev, zz, s);
  }
  const int dk = d / c.n_heads;
  for (int l = 0; l < L; ++l) {
    const gam_layer_weights& w = h->layers[l];
    const LayerMaps& m = h->lmaps[l];
    // x += 0.5 * FF1(LN(x))                                     (encoder.py:480-483)
    { PROF(PC_GEMM_FFN_UP);
      rc |= launch_gemm(GEMM_BIAS_SILU_F16, &p->m_a16, &m.ff1_w1, R, c.d_ff, d, w.ff1_b1, nullptr, p->big16, c.d_ff, 1.f, ncl, s, 0, rdev,
                        &p->o_hid); }
    { PROF(PC_GEMM_FFN_DOWN);
      rc |= launch_gemm(GEMM_BIAS_RES_F32, &p->m_hid, &m.ff1_w2, R, d, c.d_ff, w.ff1_b2, p->x, p->x, d, 0.5f, ncl, s, zz, rdev); }
    // x += W_o attn(q = W_q rope(u), k = W_k rope(u), v = W_v u), u = LN(x)   (encoder.py:485-487, 236-277)
    if (c.self_attention == 0) {
      { PROF(PC_LAYERNORM);
        launch_ln_rope_f16(p->x, w.ln_att_g, w.ln_att_b, h->w.rope_cos, h->w.rope_sin, p->a16, p->r16, R, rdev, p->row_t, p->T2,
                           dk / 2, 0, s); }
      bool merged = false;
      if (m.qkv_merged) {
        PROF(PC_GEMM_QKV);
        merged = launch_gemm_dual_a(&p->m_r16, &p->m_a16, 2 * d, &m.w_qkv, R, 3 * d, d, w.b_qk, p->big16, 3 * d, ncl, s, zz, rdev,
                                    &p->o_qkv) == 0;
      }
      if (!merged) {
        { PROF(PC_GEMM_QKV);
          rc |= launch_gemm(GEMM_BIAS_F16, &p->m_r16, &m.w_qk, R, 2 * d, d, w.b_qk, nullptr, p->big16, 3 * d, 1.f, ncl, s, zz, rdev,
                            &p->o_qk); }
        { PROF(PC_GEMM_QKV);
          rc |= launch_gemm(GEMM_BIAS_F16, &p->m_a16, &m.w_v, R, d, d, w.b_v, nullptr, p->big16 + 2 * d, 3 * d, 1.f, ncl, s, zz, rdev,
                            &p->o_v); }
      }
      { PROF(PC_ATTENTION);
        rc |= launch_attention(&p->m_qkv, p->plen, p->cu, p->o16, B, p->T2, c.n_heads, dk, d, s); }
    } else {
      // rel_pos (encoder.py:208-228): one projection GEMM -> [q+u | q+v | k | v], position scores inside the kernel
      { PROF(PC_LAYERNORM);
        launch_ln_f16(p->x, w.ln_att_g, w.ln_att_b, p->a16, R, rdev, 0, s); }
      { PROF(PC_GEMM_QKV);
        rc |= launch_gemm(GEMM_BIAS_F16, &p->m_a16, &m.w_qkv_rel, R, 4 * d, d, w.b_qkv_rel, nullptr, p->big16, 4 * d, 1.f, ncl, s, zz, rdev,
                          &p->o_qkv4); }
      { PROF(PC_ATTENTION);
        rc |= launch_attention_relpos(&p->m_qkv4, &m.pos_proj, h->max_t, p->plen, p->cu, p->o16, B, p->T2, c.n_heads, dk, d, s); }
    }
    { PROF(PC_GEMM_PROJ);
      rc |= launch_gemm(GEMM_BIAS_RES_F32, &p->m_o16, &m.w_o, R, d, d, w.b_o, p->x, p->x, d, 1.f, ncl, s, zz, rdev); }
    // x += Conv(LN(x))                                           (encoder.py:489-491, 396-409)
    { PROF(PC_LAYERNORM);
      launch_ln_f16(p->x, w.ln_conv_g, w.ln_conv_b, p->a16, R, rdev, 0, s); }
    { PROF(PC_GEMM_GLU);
      rc |= launch_gemm(GEMM_BIAS_GLU_F16, &p->m_a16, &m.pw1, R, 2 * d, d, w.pw1_b, nullptr, p->g16, d, 1.f, ncl, s, zz, rdev, &p->o_g16); }
    { PROF(PC_DWCONV);
      if (c.conv_norm == 0)
        rc |= launch_dwconv_bn_silu(p->g16, w.dw_w, w.dw_b, p->len2, p->cu, p->plen, p->o16, B, p->T2, c.conv_kernel_size, s);
      else
        rc |= launch_dwconv_ln_silu(p->g16, w.dw_w, w.dw_b, w.cn_g, w.cn_b, p->len2, p->cu, p->row_b, p->row_t, rdev, p->o16, B, p->T2,
                                    c.conv_kernel_size, s); }
    { PROF(PC_GEMM_PROJ);
      rc |= launch_gemm(GEMM_BIAS_RES_F32, &p->m_o16, &m.pw2, R, d, d, w.pw2_b, p->x, p->x, d, 1.f, ncl, s, zz, rdev); }
    // x += 0.5 * FF2(LN(x))                                      (encoder.py:493-495)
    { PROF(PC_LAYERNORM);
      launch_ln_f16(p->x, w.ln_ff2_g, w.ln_ff2_b, p->a16, R, rdev, 0, s); }
    { PROF(PC_GEMM_FFN_UP);
      rc |= launch_gemm(GEMM_BIAS_SILU_F16, &p->m_a16, &m.ff2_w1, R, c.d_ff, d, w.ff2_b1, nullptr, p->big16, c.d_ff, 1.f, ncl, s, zz, rdev,
                        &p->o_hid); }
    { PROF(PC_GEMM_FFN_DOWN);
      rc |= launch_gemm(GEMM_BIAS_RES_F32, &p->m_hid, &m.ff2_w2, R, d, c.d_ff, w.ff2_b2, p->x, p->x, d, 0.5f, ncl, s, 0, rdev); }
    // x = LN_out(x) (+ next layer's first LN fused)                (encoder.py:497)
    { PROF(PC_LAYERNORM);
      if (l + 1 < L)
        launch_ln_out_ln(p->x, w.ln_out_g, w.ln_out_b, h->layers[l + 1].ln_ff1_g, h->layers[l + 1].ln_ff1_b, p->x, p->a16, R, rdev, zz, s);
      else   // last layer: norm_out straight into the caller's padded [B, T', d] (frames that do not exist -> 0)
        launch_unpack_rows(p->x, w.ln_out_g, w.ln_out_b, p->cu, p->plen, enc, B, p->T2, zz, s); }
    if (rc) return fail(h, -4, "layer %d: a launch was rejected (rc=%d): %s", l, rc, cudaGetErrorString(cudaGetLastError()));
  }
  cudaMemcpyAsync(enc_len, p->len2, B * sizeof(int), cudaMemcpyDeviceToDevice, s);
  GAM_CHECK_LAUNCH(h, "encode");
  return 0;
}

// ---- the heads.  Each workspace has one layout, which both its size query (for the greedy decoders, the launcher's size
// check) and its carve follow; and the joint's projections, shared by its forward, alignment, backward and loss entry points.
namespace {
// greedy decoding: CTC, the label of every row (and, scored, its l); RNN-T, the encoder projection of every row.  Returns where
// the last piece ends, the least each launcher accepts; gam_decode_*workspace_bytes size for either head.
struct DecodeWs { int* labels; float *lp, *encproj; };
int64_t decode_layout(const gam_config& c, int64_t R, bool scored, uint8_t* base, DecodeWs* w) {
  Carve cv{base};
  w->labels = c.head == 1 ? cv.take<int>(R) : nullptr;
  w->lp = c.head == 1 && scored ? cv.take(R) : nullptr;
  w->encproj = c.head == 2 ? cv.take(R * c.joint_hidden) : nullptr;
  return cv.end;
}

// the checks of gam_ctc_align and gam_rnnt_align(_scores): the head, and T and U within the short-form limits
int align_args(gam_handle* h, const char* what, int head, int32_t B, int32_t T, int32_t U) {
  if (h->cfg.head != head) return fail(h, -1, "%s: model has no %s head", what, head == 1 ? "CTC" : "RNN-T");
  if (B <= 0 || T <= 0 || U < 0) return fail(h, -1, "%s: bad sizes (B=%d, T=%d, U=%d)", what, B, T, U);
  if (T > h->max_t) return fail(h, -1, "%s: T=%d exceeds the handle's max_encoded_frames %d", what, T, h->max_t);
  if (U > kAlignMaxTokens) return fail(h, -1, "%s: U=%d exceeds %d tokens per utterance", what, U, kAlignMaxTokens);
  return 0;
}

// CTC alignment: the backpointers, and with gaps m[t] of every frame behind them
struct CtcAlignWs { uint32_t* bp; float* m; };
int64_t ctc_align_layout(int32_t B, int32_t T, int32_t U, bool gaps, uint8_t* base, CtcAlignWs* w) {
  Carve cv{base};
  w->bp = cv.take<uint32_t>(static_cast<int64_t>(B) * ctc_bp_words(T, U));
  w->m = gaps ? cv.take(static_cast<int64_t>(B) * T) : nullptr;
  return cv.off;
}

constexpr int64_t kProjMaxRows = 65535LL * 64;   // grid.y limit of the projection GEMMs (64 rows per block)

// what every joint entry point needs: at most kProjMaxRows rows in each projection, pred_hidden and d_model multiples of 16
bool proj_shapes_ok(const gam_config& c, int32_t B, int32_t T, int32_t U1) {
  return static_cast<int64_t>(B) * T <= kProjMaxRows && static_cast<int64_t>(B) * U1 <= kProjMaxRows && c.pred_hidden % 16 == 0 &&
         c.d_model % 16 == 0;
}

// ... and, for the forward joint kernels (hidden_tile), the hidden tile in shared memory
int joint_args(gam_handle* h, const char* what, int32_t B, int32_t T, int32_t U1, bool hidden_tile) {
  const int J = h->cfg.joint_hidden;
  if (hidden_tile && (J % 4 != 0 || J > rnnt_joint_max_hidden()))
    return fail(h, -1, "%s: needs joint_hidden %% 4 == 0 and <= %d (joint_hidden %d)", what, rnnt_joint_max_hidden(), J);
  if (proj_shapes_ok(h->cfg, B, T, U1)) return 0;
  return fail(h, -1, "%s: needs B*T and B*U <= %lld, pred_hidden %% 16 == 0 and d_model %% 16 == 0 (B=%d, T=%d, %d decoder rows, "
              "pred_hidden %d)", what, (long long)kProjMaxRows, B, T, U1, h->cfg.pred_hidden);
}

// E = enc W_e^T + b_e [B*T, J] and P = dec W_p + b_p [B*U1, J], one launch each
void rnnt_project(gam_handle* h, const float* enc, const float* dec, int32_t B, int32_t T, int32_t U1, float* E, float* P,
                  int prof_class, cudaStream_t s) {
  const gam_config& c = h->cfg;
  { PROF(prof_class);
    launch_sgemm_tn_bias(enc, h->w.rnnt_enc_w, h->w.rnnt_enc_b, E, B * T, c.joint_hidden, c.d_model, s); }
  { PROF(prof_class);
    launch_sgemm_nn_bias(dec, h->w.rnnt_wp_t, h->w.rnnt_bp, P, B * U1, c.joint_hidden, c.pred_hidden, s); }
}

// gam_rnnt_joint's and gam_rnnt_align_scores' workspace: the two projections
struct ProjWs { float *E, *P; };
int64_t proj_layout(const gam_config& c, int32_t B, int32_t T, int32_t U1, uint8_t* base, ProjWs* w) {
  Carve cv{base};
  w->E = cv.take(static_cast<int64_t>(B) * T * c.joint_hidden);
  w->P = cv.take(static_cast<int64_t>(B) * U1 * c.joint_hidden);
  return cv.off;
}

inline int64_t max3(int64_t a, int64_t b, int64_t c) { return a > b ? (a > c ? a : c) : (b > c ? b : c); }

struct CtcBwdWs { float *dl, *part; };
int64_t ctc_bwd_layout(const gam_config& c, int64_t R, uint8_t* base, CtcBwdWs* w) {
  Carve cv{base};
  w->dl = cv.take(R * c.num_classes);
  w->part = cv.take(outer_sum_workspace_floats(R, c.num_classes, c.d_model, true));
  return cv.off;
}

struct JointBwdWs { float *E, *P, *dl, *dhid, *dE, *dP, *part; };
int64_t joint_bwd_layout(const gam_config& c, int32_t B, int32_t T, int32_t U, uint8_t* base, JointBwdWs* w) {
  const int64_t J = c.joint_hidden, BT = static_cast<int64_t>(B) * T, BU = static_cast<int64_t>(B) * U, rows = BT * U;
  Carve cv{base};
  w->E = cv.take(BT * J);
  w->P = cv.take(BU * J);
  w->dl = cv.take(rows * c.num_classes);
  w->dhid = cv.take(rows * J);
  w->dE = cv.take(BT * J);
  w->dP = cv.take(BU * J);
  w->part = cv.take(max3(outer_sum_workspace_floats(rows, c.num_classes, J, true), outer_sum_workspace_floats(BT, J, c.d_model, true),
                         outer_sum_workspace_floats(BU, J, c.pred_hidden, true)));
  return cv.off;
}

struct PredBwdWs { float *dgates, *dcc, *dcls, *part; };
int64_t pred_bwd_layout(const gam_config& c, int32_t B, int32_t U, uint8_t* base, PredBwdWs* w) {
  const int64_t H = c.pred_hidden, BU = static_cast<int64_t>(B) * U;
  Carve cv{base};
  w->dgates = cv.take(BU * 4 * H);
  w->dcc = cv.take(static_cast<int64_t>(B) * H);
  w->dcls = cv.take(static_cast<int64_t>(c.num_classes) * 4 * H);
  w->part = cv.take(max3(outer_sum_workspace_floats(BU, 4 * H, H, true), outer_sum_workspace_floats(c.num_classes, 4 * H, H, false), 0));
  return cv.off;
}

// the gradients of the joint's inputs from dE [BT, J] and dP [BU, J], each optional (a weight gradient with its bias): dW_enc /
// db_enc and dW_pred / db_pred (part: the outer sums' partials), d_enc = dE W_e and d_dec = dP W_p
void joint_input_grads(gam_handle* h, const float* enc, const float* dec, int64_t BT, int64_t BU, const float* dE, const float* dP,
                       float* part, float* d_enc, float* d_dec, float* dW_enc, float* db_enc, float* dW_pred, float* db_pred,
                       cudaStream_t s) {
  const gam_config& c = h->cfg;
  const int J = c.joint_hidden;
  if (dW_enc != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_outer_sum(dE, enc, BT, J, c.d_model, dW_enc, db_enc, part, s); }
  if (dW_pred != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_outer_sum(dP, dec, BU, J, c.pred_hidden, dW_pred, db_pred, part, s); }
  if (d_enc != nullptr) { PROF(PC_HEAD_BACKWARD);   // W_e [J, d]
    launch_head_matmul(dE, h->w.rnnt_enc_w, c.d_model, 1, d_enc, BT, J, c.d_model, nullptr, nullptr, 1, 1, s); }
  if (d_dec != nullptr) { PROF(PC_HEAD_BACKWARD);   // W_p [J, H] = rnnt_wp_t^T
    launch_head_matmul(dP, h->w.rnnt_wp_t, 1, J, d_dec, BU, J, c.pred_hidden, nullptr, nullptr, 1, 1, s); }
}

bool loss_sizes_ok(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || T <= 0 || T > h->max_t || U < 0 || U > kAlignMaxTokens) return false;
  const int J = h->cfg.joint_hidden;
  return J % 4 == 0 && J <= rnnt_joint_max_hidden() && J <= rnnt_loss_max_hidden() && proj_shapes_ok(h->cfg, B, T, U + 1);
}

int loss_args(gam_handle* h, const char* what, int32_t B, int32_t T, int32_t U) {
  if (h->cfg.head != 2) return fail(h, -1, "%s: model has no RNN-T head", what);
  if (loss_sizes_ok(h, B, T, U)) return 0;
  return fail(h, -1, "%s: unsupported sizes (B=%d, T=%d, U=%d; T <= %d, U <= %d, joint_hidden %d <= %d)", what, B, T, U, h->max_t,
              kAlignMaxTokens, h->cfg.joint_hidden, rnnt_loss_max_hidden());
}

struct LossFwdWs { float *E, *P, *blank, *label, *alpha; };
int64_t loss_fwd_layout(const gam_config& c, int32_t B, int32_t T, int32_t U, uint8_t* base, LossFwdWs* w) {
  const int64_t J = c.joint_hidden, BT = static_cast<int64_t>(B) * T, BU1 = static_cast<int64_t>(B) * (U + 1), N = BT * (U + 1);
  Carve cv{base};
  w->E = cv.take(BT * J);
  w->P = cv.take(BU1 * J);
  w->blank = cv.take(N);
  w->label = cv.take(N);
  w->alpha = cv.take(N);
  return cv.off;
}

struct LossBwdWs { float *E, *P, *dE, *dP, *dE_part, *dP_part, *part; };
int64_t loss_bwd_layout(const gam_config& c, int32_t B, int32_t T, int32_t U, uint8_t* base, LossBwdWs* w) {
  const RnntLossPlan p = rnnt_loss_plan(B, T, U, c.num_classes);
  const int64_t J = c.joint_hidden, BT = static_cast<int64_t>(B) * T, BU1 = static_cast<int64_t>(B) * (U + 1);
  Carve cv{base};
  w->E = cv.take(BT * J);
  w->P = cv.take(BU1 * J);
  w->dE = cv.take(BT * J);
  w->dP = cv.take(BU1 * J);
  w->dE_part = cv.take(p.NS * BT * J);
  w->dP_part = cv.take(p.ST * BU1 * J);
  w->part = cv.take(max3(p.S > 1 ? static_cast<int64_t>(p.S) * c.num_classes * (J + 1) : 0,
                         outer_sum_workspace_floats(BT, static_cast<int>(J), c.d_model, true),
                         outer_sum_workspace_floats(BU1, static_cast<int>(J), c.pred_hidden, true)));
  return cv.off;
}
}  // namespace

// the greedy decoders' launches, after each entry point's own checks: labels and (scored) l of every row in the workspace,
// then the collapse (io: a fresh or a resume call, kernels.h)
static int ctc_greedy_impl(gam_handle* h, const char* what, const float* enc, int32_t B, int32_t T, void* workspace,
                           const GreedyIo& io, void* stream) {
  const gam_config& c = h->cfg;
  const int64_t R = static_cast<int64_t>(B) * T;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DecodeWs w;
  decode_layout(c, R, io.token_logp != nullptr, static_cast<uint8_t*>(workspace), &w);
  { PROF(PC_CTC_ARGMAX);
    launch_ctc_argmax(enc, h->w.ctc_w, h->w.ctc_b, w.labels, w.lp, static_cast<int>(R), c.d_model, c.num_classes, s); }
  { PROF(PC_CTC_COLLAPSE);
    launch_ctc_collapse(w.labels, w.lp, B, T, c.num_classes - 1, io, s); }
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

// the encoder projection of every row into the workspace, then the cluster kernel (boosted unless boost is NULL)
static int rnnt_greedy_impl(gam_handle* h, const char* what, const float* enc, int32_t B, int32_t T, void* workspace,
                            const GreedyIo& io, void* stream, const BoostGraph* boost = nullptr) {
  const gam_config& c = h->cfg;
  const int64_t R = static_cast<int64_t>(B) * T;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DecodeWs w;
  decode_layout(c, R, false, static_cast<uint8_t*>(workspace), &w);
  { PROF(PC_RNNT_ENCPROJ);   // a row's projection does not depend on the others, so a resume call projects every row too
    launch_sgemm_tn_bias(enc, h->w.rnnt_enc_w, h->w.rnnt_enc_b, w.encproj, static_cast<int>(R), c.joint_hidden, c.d_model, s); }
  PROF(PC_RNNT_GREEDY);
  const int rc = launch_rnnt_greedy(w.encproj, h->w.rnnt_emb_gates, h->w.rnnt_whh_t, h->w.rnnt_wp_t, h->w.rnnt_bp, h->w.rnnt_wo,
                                    h->w.rnnt_bo, B, T, c.pred_hidden, c.num_classes, c.num_classes - 1, c.max_symbols, io, boost,
                                    nullptr, s);
  if (rc > 0)
    return fail(h, -1, "rnnt: the greedy kernel is specialised for pred_hidden = joint_hidden = 320 and needs 16-CTA clusters "
                "(pred_hidden %d)", c.pred_hidden);
  if (rc < 0) return fail(h, -4, "rnnt cluster kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

// a one-shot call: every row from a fresh stream over [0, enc_len[b])
static GreedyIo fresh_io(const int32_t* enc_len, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp,
                         float* path_logp, int32_t* path_rows) {
  GreedyIo io{};
  io.ids = ids; io.frames = frames; io.counts = counts; io.max_out = max_out;
  io.token_logp = token_logp; io.path_logp = path_logp; io.path_rows = path_rows;
  io.hi = enc_len;
  return io;
}

int gam_ctc_greedy(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                   int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 1) return fail(h, -1, "model has no CTC head");
  if (max_out < T) return fail(h, -1, "max_out (%d) must be >= T (%d)", max_out, T);
  if (max_out != T) return fail(h, -1, "ids/frames row pitch must equal T for the CTC path");
  DecodeWs w;
  if (workspace_bytes < decode_layout(c, static_cast<int64_t>(B) * T, false, nullptr, &w))
    return fail(h, -1, "workspace too small for CTC labels");
  return ctc_greedy_impl(h, "ctc_greedy", enc, B, T, workspace,
                         fresh_io(enc_len, ids, frames, counts, max_out, nullptr, nullptr, nullptr), stream);
}

int gam_ctc_greedy_scored(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                          int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                          float* token_logp, float* path_logp, int32_t* path_rows, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 1) return fail(h, -1, "model has no CTC head");
  if (max_out < T) return fail(h, -1, "max_out (%d) must be >= T (%d)", max_out, T);
  if (max_out != T) return fail(h, -1, "ids/frames row pitch must equal T for the CTC path");
  if (!token_logp || !path_logp || !path_rows) return fail(h, -1, "ctc_greedy_scored: token_logp, path_logp and path_rows are required");
  DecodeWs w;
  if (workspace_bytes < decode_layout(c, static_cast<int64_t>(B) * T, true, nullptr, &w))
    return fail(h, -1, "workspace too small for CTC labels and scores");
  return ctc_greedy_impl(h, "ctc_greedy_scored", enc, B, T, workspace,
                         fresh_io(enc_len, ids, frames, counts, max_out, token_logp, path_logp, path_rows), stream);
}

static int rnnt_greedy_args(gam_handle* h, int32_t B, int32_t T, int64_t workspace_bytes) {
  const gam_config& c = h->cfg;
  if (c.head != 2) return fail(h, -1, "model has no RNN-T head");
  if (c.pred_hidden != c.joint_hidden) return fail(h, -1, "pred_hidden != joint_hidden is not supported");
  DecodeWs w;
  if (workspace_bytes < decode_layout(c, static_cast<int64_t>(B) * T, false, nullptr, &w))
    return fail(h, -1, "workspace too small for the RNN-T encoder projection");
  return 0;
}

int gam_rnnt_greedy_scored(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                           int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out,
                           float* token_logp, float* path_logp, int32_t* path_rows, void* stream) {
  if (!token_logp || !path_logp || !path_rows) return fail(h, -1, "rnnt_greedy_scored: token_logp, path_logp and path_rows are required");
  if (rnnt_greedy_args(h, B, T, workspace_bytes) != 0) return -1;
  return rnnt_greedy_impl(h, "rnnt_greedy", enc, B, T, workspace,
                          fresh_io(enc_len, ids, frames, counts, max_out, token_logp, path_logp, path_rows), stream);
}

int gam_rnnt_greedy(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                    int64_t workspace_bytes, int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out, void* stream) {
  if (rnnt_greedy_args(h, B, T, workspace_bytes) != 0) return -1;
  return rnnt_greedy_impl(h, "rnnt_greedy", enc, B, T, workspace,
                          fresh_io(enc_len, ids, frames, counts, max_out, nullptr, nullptr, nullptr), stream);
}

int64_t gam_decode_state_bytes(const gam_handle* h) {
  if (h->cfg.head == 1) return kCtcDecodeStateBytes;
  if (h->cfg.head == 2) return kRnntDecodeStateBytes;
  return -1;
}

int gam_decode_state_init(gam_handle* h, void* state, int32_t n, void* stream) {
  const int64_t bytes = gam_decode_state_bytes(h);
  if (bytes < 0) return fail(h, -1, "decode_state_init: model has no CTC or RNN-T head");
  if (n < 0 || (n > 0 && state == nullptr)) return fail(h, -1, "decode_state_init: bad state buffer (n=%d)", n);
  launch_decode_state_init(static_cast<uint8_t*>(state), bytes, n, h->cfg.num_classes - 1, static_cast<cudaStream_t>(stream));
  GAM_CHECK_LAUNCH(h, "decode_state_init");
  return 0;
}

int64_t gam_decode_resume_workspace_bytes(const gam_handle* h, int32_t B, int32_t T) {
  return gam_decode_scored_workspace_bytes(h, B, T);
}

// shared argument checks of gam_*_greedy_resume
static int resume_args(gam_handle* h, const char* what, int head, const float* enc, int32_t B, int32_t T, const int32_t* lo,
                       const int32_t* hi, const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes,
                       int32_t* ids, int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp,
                       int32_t* path_rows, double* frame_logp, int32_t* frame_rows, int64_t frame_pitch) {
  if (h->cfg.head != head) return fail(h, -1, "%s: model has no %s head", what, head == 1 ? "CTC" : "RNN-T");
  if (B < 1 || T < 1 || static_cast<int64_t>(B) * T > INT32_MAX) return fail(h, -1, "%s: bad sizes (B=%d, T=%d)", what, B, T);
  if (max_out < 1) return fail(h, -1, "%s: max_out (%d) must be >= 1", what, max_out);
  if (!enc || !lo || !hi || !frame_base || !state || !ids || !frames || !counts)
    return fail(h, -1, "%s: enc, lo, hi, frame_base, state, ids, frames and counts are required", what);
  if (token_logp && (!path_logp || !path_rows || !frame_logp || !frame_rows || frame_pitch < 1))
    return fail(h, -1, "%s: a scored call needs path_logp, path_rows, frame_logp, frame_rows and frame_pitch >= 1", what);
  return workspace_base(h, what, workspace, workspace_bytes, gam_decode_resume_workspace_bytes(h, B, T), false) ? 0 : -1;
}

// a resume call: stream b continues from its DecodeState over [lo[b], hi[b])
static GreedyIo resume_io(const int32_t* lo, const int32_t* hi, const int32_t* frame_base, void* state, int64_t stride, int32_t* ids,
                          int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                          double* frame_logp, int32_t* frame_rows, int64_t frame_pitch) {
  GreedyIo io = fresh_io(hi, ids, frames, counts, max_out, token_logp, path_logp, path_rows);
  io.frame_logp = frame_logp; io.frame_rows = frame_rows; io.frame_pitch = frame_pitch;
  io.lo = lo; io.frame_base = frame_base; io.state = static_cast<uint8_t*>(state); io.stride = stride;
  return io;
}

int gam_ctc_greedy_resume(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                          const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                          int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                          double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, void* stream) {
  if (resume_args(h, "ctc_greedy_resume", 1, enc, B, T, lo, hi, frame_base, state, workspace, workspace_bytes, ids, frames, counts,
                  max_out, token_logp, path_logp, path_rows, frame_logp, frame_rows, frame_pitch) != 0)
    return -1;
  // the ranges live on the device, so every row is labelled; each row's label and l do not depend on the others
  return ctc_greedy_impl(h, "ctc_greedy_resume", enc, B, T, workspace,
                         resume_io(lo, hi, frame_base, state, kCtcDecodeStateBytes, ids, frames, counts, max_out, token_logp,
                                   path_logp, path_rows, frame_logp, frame_rows, frame_pitch), stream);
}

static int rnnt_resume(gam_handle* h, const char* what, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                       const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids, int32_t* frames,
                       int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows, double* frame_logp,
                       int32_t* frame_rows, int64_t frame_pitch, void* stream, const BoostGraph* boost) {
  if (resume_args(h, what, 2, enc, B, T, lo, hi, frame_base, state, workspace, workspace_bytes, ids, frames, counts, max_out,
                  token_logp, path_logp, path_rows, frame_logp, frame_rows, frame_pitch) != 0)
    return -1;
  if (h->cfg.pred_hidden != h->cfg.joint_hidden) return fail(h, -1, "pred_hidden != joint_hidden is not supported");
  return rnnt_greedy_impl(h, what, enc, B, T, workspace,
                          resume_io(lo, hi, frame_base, state, kRnntDecodeStateBytes, ids, frames, counts, max_out, token_logp,
                                    path_logp, path_rows, frame_logp, frame_rows, frame_pitch), stream, boost);
}

int gam_rnnt_greedy_resume(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                           const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                           int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                           double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, void* stream) {
  return rnnt_resume(h, "rnnt_greedy_resume", enc, B, T, lo, hi, frame_base, state, workspace, workspace_bytes, ids, frames, counts,
                     max_out, token_logp, path_logp, path_rows, frame_logp, frame_rows, frame_pitch, stream, nullptr);
}

// the boost graph's own checks (gam_rnnt_greedy_boost, gam_test_rnnt_greedy_boost)
static bool boost_args(gam_handle* h, const char* what, const int32_t* next, const float* bonus, int32_t n_states, BoostGraph* g) {
  if (!next || !bonus) { fail(h, -1, "%s: boost_next and boost_bonus are required", what); return false; }
  if (n_states < 1 || n_states > kBoostMaxStates) {
    fail(h, -1, "%s: n_states (%d) must be in [1, %d]", what, n_states, kBoostMaxStates);
    return false;
  }
  *g = BoostGraph{next, bonus, n_states};
  return true;
}

int gam_rnnt_greedy_boost(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                          const int32_t* frame_base, void* state, void* workspace, int64_t workspace_bytes, int32_t* ids,
                          int32_t* frames, int32_t* counts, int32_t max_out, float* token_logp, float* path_logp, int32_t* path_rows,
                          double* frame_logp, int32_t* frame_rows, int64_t frame_pitch, const int32_t* boost_next,
                          const float* boost_bonus, int32_t n_states, void* stream) {
  if (h->cfg.head != 2) return fail(h, -1, "rnnt_greedy_boost: model has no RNN-T head");
  BoostGraph g;
  if (!boost_args(h, "rnnt_greedy_boost", boost_next, boost_bonus, n_states, &g)) return -1;
  return rnnt_resume(h, "rnnt_greedy_boost", enc, B, T, lo, hi, frame_base, state, workspace, workspace_bytes, ids, frames, counts,
                     max_out, token_logp, path_logp, path_rows, frame_logp, frame_rows, frame_pitch, stream, &g);
}

int gam_ctc_log_probs(gam_handle* h, const float* enc, int32_t B, int32_t T, float* log_probs, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 1) return fail(h, -1, "ctc_log_probs: model has no CTC head");
  if (B <= 0 || T <= 0) return fail(h, -1, "ctc_log_probs: bad sizes (B=%d, T=%d)", B, T);
  const int64_t R = static_cast<int64_t>(B) * T;
  if (R > INT32_MAX) return fail(h, -1, "ctc_log_probs: B*T = %lld exceeds 2^31 - 1 frames", (long long)R);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_CTC_LOG_PROBS);
    launch_ctc_log_probs(enc, h->w.ctc_w, h->w.ctc_b, log_probs, static_cast<int>(R), c.d_model, c.num_classes, s); }
  GAM_CHECK_LAUNCH(h, "ctc_log_probs");
  return 0;
}

// ---- the RNN-T joint lattice
int64_t gam_rnnt_joint_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || T <= 0 || U <= 0) return -1;
  ProjWs w;
  return proj_layout(h->cfg, B, T, U, nullptr, &w) + 1024;
}

int gam_rnnt_joint(gam_handle* h, const float* enc, const float* dec, int32_t B, int32_t T, int32_t U, void* workspace,
                   int64_t workspace_bytes, float* out, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 2) return fail(h, -1, "rnnt_joint: model has no RNN-T head");
  if (B <= 0 || T <= 0 || U <= 0) return fail(h, -1, "rnnt_joint: bad sizes (B=%d, T=%d, U=%d)", B, T, U);
  if (joint_args(h, "rnnt_joint", B, T, U, true) != 0) return -1;
  uint8_t* ws = workspace_base(h, "rnnt_joint", workspace, workspace_bytes, gam_rnnt_joint_workspace_bytes(h, B, T, U), true);
  if (!ws) return -1;
  ProjWs w;
  proj_layout(c, B, T, U, ws, &w);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rnnt_project(h, enc, dec, B, T, U, w.E, w.P, PC_RNNT_JOINT, s);
  int rc;
  { PROF(PC_RNNT_JOINT);
    rc = launch_rnnt_joint(w.E, w.P, h->w.rnnt_wo, h->w.rnnt_bo, out, B, T, U, c.joint_hidden, c.num_classes, s); }
  if (rc != 0) return fail(h, -4, "rnnt_joint: lattice launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "rnnt_joint");
  return 0;
}

// ---- alignment of known transcripts (csrc/align.cu; stage 1 of RNN-T: the gathered joint of heads.cu)
int64_t gam_ctc_align_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 1 || B <= 0 || T <= 0 || T > h->max_t || U < 0 || U > kAlignMaxTokens) return -1;
  CtcAlignWs w;
  return ctc_align_layout(B, T, U, false, nullptr, &w);
}

int gam_ctc_align(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets, const int32_t* target_len,
                  int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                  float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream) {
  const gam_config& c = h->cfg;
  if (align_args(h, "ctc_align", 1, B, T, U) != 0) return -1;
  if (!log_probs || !enc_len || !target_len || (U > 0 && (!targets || !frames || !token_logp)) || !viterbi_logp || !log_likelihood ||
      !path_rows)
    return fail(h, -1, "ctc_align: a required pointer is NULL");
  uint8_t* ws = workspace_base(h, "ctc_align", workspace, workspace_bytes, gam_ctc_align_workspace_bytes(h, B, T, U), false);
  if (!ws) return -1;
  CtcAlignWs w;
  ctc_align_layout(B, T, U, false, ws, &w);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_ALIGN);
    rc = launch_ctc_align(log_probs, enc_len, targets, target_len, B, T, U, c.num_classes, w.bp, frames, token_logp, viterbi_logp,
                          log_likelihood, path_rows, s); }
  if (rc != 0) return fail(h, -4, "ctc_align: launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "ctc_align");
  return 0;
}

int64_t gam_ctc_align_long_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 1 || B <= 0 || T <= 0 || U < 0 || U > kAlignLongMaxTokens) return -1;
  CtcAlignWs w;
  return ctc_align_layout(B, T, U, false, nullptr, &w);
}

int64_t gam_ctc_align_long_gaps_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (gam_ctc_align_long_workspace_bytes(h, B, T, U) < 0) return -1;
  CtcAlignWs w;
  return ctc_align_layout(B, T, U, true, nullptr, &w);
}

// gaps: NULL for gam_ctc_align_long; otherwise line_edges, log_theta and the three outputs, with m still to be placed in the
// workspace behind the backpointers
static int ctc_align_long_run(gam_handle* h, const char* what, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                              const int32_t* target_len, int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes,
                              int32_t* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int32_t* path_rows,
                              int32_t cluster_ctas, int32_t* plan, AlignGaps* gaps, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 1) return fail(h, -1, "%s: model has no CTC head", what);
  if (B <= 0 || T <= 0 || U < 0) return fail(h, -1, "%s: bad sizes (B=%d, T=%d, U=%d)", what, B, T, U);
  if (U > kAlignLongMaxTokens) return fail(h, -1, "%s: U=%d exceeds %d tokens per utterance", what, U, kAlignLongMaxTokens);
  if (static_cast<int64_t>(B) * kAlignLongMaxCtas > INT32_MAX) return fail(h, -1, "%s: B=%d is too large", what, B);
  if (!log_probs || !enc_len || !target_len || (U > 0 && (!targets || !frames || !token_logp)) || !viterbi_logp || !log_likelihood ||
      !path_rows)
    return fail(h, -1, "%s: a required pointer is NULL", what);
  if (gaps) {
    if ((U > 0 && !gaps->line_edges) || !gaps->unmatched || !gaps->unmatched_rows || !gaps->unmatched_logp)
      return fail(h, -1, "%s: a required pointer is NULL", what);
    if (std::isnan(gaps->log_theta) || gaps->log_theta > 0.f)
      return fail(h, -1, "%s: log_theta=%g must be <= 0 (a threshold in (0, 1]) or -inf", what, gaps->log_theta);
    if (gaps->skipped_rows) {
      if (!gaps->skip_logp) return fail(h, -1, "%s: a required pointer is NULL", what);
      if (std::isnan(gaps->log_psi) || gaps->log_psi > 0.f)
        return fail(h, -1, "%s: log_psi=%g must be <= 0 (a threshold in (0, 1]) or -inf", what, gaps->log_psi);
    }
  }
  const int64_t need = gaps ? gam_ctc_align_long_gaps_workspace_bytes(h, B, T, U) : gam_ctc_align_long_workspace_bytes(h, B, T, U);
  uint8_t* ws = workspace_base(h, what, workspace, workspace_bytes, need, false);
  if (!ws) return -1;
  CtcAlignWs w;
  ctc_align_layout(B, T, U, gaps != nullptr, ws, &w);
  if (gaps) gaps->m = w.m;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_ALIGN);
    if (gaps) h->launches += 1;   // the pre-pass
    rc = launch_ctc_align_long(log_probs, enc_len, targets, target_len, B, T, U, c.num_classes, cluster_ctas, w.bp, frames, token_logp,
                               viterbi_logp, log_likelihood, path_rows, plan, gaps, s); }
  if (rc == 2) return fail(h, -1, "%s: %d CTAs leave a CTA without states at U=%d", what, cluster_ctas, U);
  if (rc == 1) return fail(h, -1, "%s: no cluster of <= %d CTAs holds U=%d (forced %d)", what, kAlignLongMaxCtas, U, cluster_ctas);
  if (rc != 0) return fail(h, -4, "%s: launch rejected (rc=%d): %s", what, rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

int gam_ctc_align_long(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets, const int32_t* target_len,
                       int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                       float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream) {
  return ctc_align_long_run(h, "ctc_align_long", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes, frames,
                            token_logp, viterbi_logp, log_likelihood, path_rows, 0, nullptr, nullptr, stream);
}

int gam_ctc_align_long_gaps(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                            const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                            void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp, float* viterbi_logp,
                            float* log_likelihood, int32_t* path_rows, uint8_t* unmatched, int32_t* unmatched_rows,
                            float* unmatched_logp, void* stream) {
  AlignGaps g{line_edges, log_theta, nullptr, unmatched, unmatched_rows, unmatched_logp};
  return ctc_align_long_run(h, "ctc_align_long_gaps", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes,
                            frames, token_logp, viterbi_logp, log_likelihood, path_rows, 0, nullptr, &g, stream);
}

int64_t gam_ctc_align_long_skips_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  return gam_ctc_align_long_gaps_workspace_bytes(h, B, T, U);
}

int gam_ctc_align_long_skips(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                             const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                             float log_psi, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                             float* viterbi_logp, float* log_likelihood, int32_t* path_rows, uint8_t* unmatched,
                             int32_t* unmatched_rows, float* unmatched_logp, int32_t* skipped_rows, float* skip_logp, void* stream) {
  if (!skipped_rows) return fail(h, -1, "ctc_align_long_skips: a required pointer is NULL");
  AlignGaps g{line_edges, log_theta, nullptr, unmatched, unmatched_rows, unmatched_logp, log_psi, skipped_rows, skip_logp};
  return ctc_align_long_run(h, "ctc_align_long_skips", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes,
                            frames, token_logp, viterbi_logp, log_likelihood, path_rows, 0, nullptr, &g, stream);
}

int gam_test_ctc_align_long(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                            const int32_t* target_len, int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes,
                            int32_t* frames, float* token_logp, float* viterbi_logp, float* log_likelihood, int32_t* path_rows,
                            int32_t cluster_ctas, int32_t* plan, void* stream) {
  if (cluster_ctas < 0 || cluster_ctas > kAlignLongMaxCtas)
    return fail(h, -1, "test_ctc_align_long: cluster_ctas=%d outside [0, %d]", cluster_ctas, kAlignLongMaxCtas);
  return ctc_align_long_run(h, "test_ctc_align_long", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes,
                            frames, token_logp, viterbi_logp, log_likelihood, path_rows, cluster_ctas, plan, nullptr, stream);
}

int gam_test_ctc_align_long_gaps(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                                 const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                                 void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp, float* viterbi_logp,
                                 float* log_likelihood, int32_t* path_rows, uint8_t* unmatched, int32_t* unmatched_rows,
                                 float* unmatched_logp, int32_t cluster_ctas, int32_t* plan, void* stream) {
  if (cluster_ctas < 0 || cluster_ctas > kAlignLongMaxCtas)
    return fail(h, -1, "test_ctc_align_long_gaps: cluster_ctas=%d outside [0, %d]", cluster_ctas, kAlignLongMaxCtas);
  AlignGaps g{line_edges, log_theta, nullptr, unmatched, unmatched_rows, unmatched_logp};
  return ctc_align_long_run(h, "test_ctc_align_long_gaps", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes,
                            frames, token_logp, viterbi_logp, log_likelihood, path_rows, cluster_ctas, plan, &g, stream);
}

int gam_test_ctc_align_long_skips(gam_handle* h, const float* log_probs, const int32_t* enc_len, const int32_t* targets,
                                  const int32_t* target_len, const uint8_t* line_edges, int32_t B, int32_t T, int32_t U, float log_theta,
                                  float log_psi, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                                  float* viterbi_logp, float* log_likelihood, int32_t* path_rows, uint8_t* unmatched,
                                  int32_t* unmatched_rows, float* unmatched_logp, int32_t* skipped_rows, float* skip_logp,
                                  int32_t cluster_ctas, int32_t* plan, void* stream) {
  if (cluster_ctas < 0 || cluster_ctas > kAlignLongMaxCtas)
    return fail(h, -1, "test_ctc_align_long_skips: cluster_ctas=%d outside [0, %d]", cluster_ctas, kAlignLongMaxCtas);
  if (!skipped_rows) return fail(h, -1, "test_ctc_align_long_skips: a required pointer is NULL");
  AlignGaps g{line_edges, log_theta, nullptr, unmatched, unmatched_rows, unmatched_logp, log_psi, skipped_rows, skip_logp};
  return ctc_align_long_run(h, "test_ctc_align_long_skips", log_probs, enc_len, targets, target_len, B, T, U, workspace, workspace_bytes,
                            frames, token_logp, viterbi_logp, log_likelihood, path_rows, cluster_ctas, plan, &g, stream);
}

// ---- keyword spotting (csrc/spot.cu)
// the checks gam_ctc_spot* and gam_ctc_bias share
static int spot_args(gam_handle* h, const char* what, int32_t B, int32_t T, int32_t K, int32_t Umax, float threshold, int32_t max_det) {
  if (h->cfg.head != 1) return fail(h, -1, "%s: model has no CTC head", what);
  if (B <= 0 || B > 65535 || T <= 0) return fail(h, -1, "%s: bad sizes (B=%d, T=%d; B <= 65535)", what, B, T);
  if (K < 1) return fail(h, -1, "%s: K=%d: at least one keyword is needed", what, K);
  if (Umax < 1 || Umax > kSpotMaxTokens) return fail(h, -1, "%s: Umax=%d outside [1, %d] tokens per keyword", what, Umax, kSpotMaxTokens);
  if (!(threshold > 0.f && threshold <= 1.f)) return fail(h, -1, "%s: threshold %g outside (0, 1]", what, static_cast<double>(threshold));
  if (max_det < 1) return fail(h, -1, "%s: max_det=%d must be >= 1", what, max_det);
  return 0;
}

static int ctc_spot_run(gam_handle* h, const char* what, const float* log_probs, const SpotResume& io, int32_t B, int32_t T,
                        const int32_t* keywords, const int32_t* keyword_len, int32_t K, int32_t Umax, float threshold, int32_t max_det,
                        int32_t* det_start, int32_t* det_end, float* det_score, int32_t* det_count, int32_t warps, void* stream) {
  const gam_config& c = h->cfg;
  if (spot_args(h, what, B, T, K, Umax, threshold, max_det) != 0) return -1;
  if (!log_probs || !io.hi || !keywords || !keyword_len || !det_start || !det_end || !det_score || !det_count)
    return fail(h, -1, "%s: a required pointer is NULL", what);
  const float log_theta = static_cast<float>(std::log(static_cast<double>(threshold)));   // correctly rounded to fp32
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_ALIGN);
    rc = launch_ctc_spot(log_probs, io, keywords, keyword_len, B, T, c.num_classes, K, Umax, log_theta, max_det, warps, det_start,
                         det_end, det_score, det_count, s); }
  if (rc == 1) return fail(h, -1, "%s: a frame of %d classes does not fit in shared memory", what, c.num_classes);
  if (rc != 0) return fail(h, -4, "%s: launch rejected (rc=%d): %s", what, rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

// a one-shot call: fresh records over [0, enc_len[b]), finished
static SpotResume spot_fresh_io(const int32_t* enc_len) {
  SpotResume io{};
  io.hi = enc_len;
  return io;
}

int64_t gam_ctc_spot_state_bytes(const gam_handle* h, int32_t Umax) {
  if (!h || h->cfg.head != 1 || Umax < 1 || Umax > kSpotMaxTokens) return -1;
  return ctc_spot_record_bytes(Umax);
}

int gam_ctc_spot_state_init(gam_handle* h, void* state, int32_t n, int32_t K, int32_t Umax, void* stream) {
  const int64_t bytes = gam_ctc_spot_state_bytes(h, Umax);
  if (bytes < 0) return fail(h, -1, "ctc_spot_state_init: no CTC head, or Umax=%d outside [1, %d]", Umax, kSpotMaxTokens);
  if (n < 0 || K < 1 || static_cast<int64_t>(n) * K > INT32_MAX || (n > 0 && state == nullptr))
    return fail(h, -1, "ctc_spot_state_init: bad state buffer (n=%d, K=%d)", n, K);
  launch_ctc_spot_state_init(static_cast<uint8_t*>(state), static_cast<int64_t>(n) * K, Umax, static_cast<cudaStream_t>(stream));
  GAM_CHECK_LAUNCH(h, "ctc_spot_state_init");
  return 0;
}

int gam_ctc_spot_resume(gam_handle* h, const float* log_probs, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi,
                        const int32_t* frame_base, const int32_t* finish, const int32_t* keywords, const int32_t* keyword_len, int32_t K,
                        int32_t Umax, float threshold, int32_t max_det, void* state, int64_t record_bytes, int32_t* det_start,
                        int32_t* det_end, float* det_score, int32_t* det_count, int32_t* pend_start, int32_t* pend_end,
                        float* pend_score, void* stream) {
  if (!lo || !hi || !frame_base || !finish || !state) return fail(h, -1, "ctc_spot_resume: lo, hi, frame_base, finish and state are required");
  if (Umax >= 1 && Umax <= kSpotMaxTokens && record_bytes != ctc_spot_record_bytes(Umax))
    return fail(h, -1, "ctc_spot_resume: record_bytes=%lld, but Umax=%d needs %lld", (long long)record_bytes, Umax,
                (long long)ctc_spot_record_bytes(Umax));
  if (!pend_start != !pend_end || !pend_start != !pend_score)
    return fail(h, -1, "ctc_spot_resume: pend_start, pend_end and pend_score go together");
  SpotResume io{lo, hi, frame_base, finish, static_cast<uint8_t*>(state), record_bytes, pend_start, pend_end, pend_score};
  return ctc_spot_run(h, "ctc_spot_resume", log_probs, io, B, T, keywords, keyword_len, K, Umax, threshold, max_det, det_start, det_end,
                      det_score, det_count, 0, stream);
}

int gam_ctc_spot(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                 const int32_t* keyword_len, int32_t K, int32_t Umax, float threshold, int32_t max_det, int32_t* det_start,
                 int32_t* det_end, float* det_score, int32_t* det_count, void* stream) {
  return ctc_spot_run(h, "ctc_spot", log_probs, spot_fresh_io(enc_len), B, T, keywords, keyword_len, K, Umax, threshold, max_det,
                      det_start, det_end, det_score, det_count, 0, stream);
}

int gam_test_ctc_spot(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                      const int32_t* keyword_len, int32_t K, int32_t Umax, float threshold, int32_t max_det, int32_t* det_start,
                      int32_t* det_end, float* det_score, int32_t* det_count, int32_t warps_per_cta, void* stream) {
  if (warps_per_cta < 0 || warps_per_cta > kSpotMaxWarps)
    return fail(h, -1, "test_ctc_spot: warps_per_cta=%d outside [0, %d]", warps_per_cta, kSpotMaxWarps);
  return ctc_spot_run(h, "test_ctc_spot", log_probs, spot_fresh_io(enc_len), B, T, keywords, keyword_len, K, Umax, threshold,
                      max_det, det_start, det_end, det_score, det_count, warps_per_cta, stream);
}

// ---- hotwords (csrc/bias.cu)
int64_t gam_ctc_bias_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t K, int32_t max_det) {
  if (!h || h->cfg.head != 1 || B <= 0 || B > 65535 || T <= 0 || K < 1 || max_det < 1) return -1;
  const int64_t words = ctc_bias_workspace_words(T, K, max_det);
  if (words < 0 || words > (int64_t(1) << 40) / B) return -1;
  return align_up(static_cast<int64_t>(B) * words * 4, 1024);
}

// the checks and launches gam_ctc_bias and gam_ctc_bias_resume share; `a` holds every pointer and size but V1 and log_theta
static int ctc_bias_run(gam_handle* h, const char* what, BiasArgs& a, float threshold, int32_t V, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  const gam_config& c = h->cfg;
  if (spot_args(h, what, a.B, a.T, a.K, a.Umax, threshold, a.max_det) != 0) return -1;
  if (a.max_out < a.T) return fail(h, -1, "%s: max_out=%d is less than T=%d", what, a.max_out, a.T);
  if (!a.flags || V != c.num_classes - 1)
    return fail(h, -1, "%s: the token flag table is missing or has %d entries, not %d", what, V, c.num_classes - 1);
  if (!a.log_probs || !a.enc_len || !a.keywords || !a.keyword_len || !a.det_start || !a.det_end || !a.det_score || !a.det_count ||
      !a.ids || !a.frames || !a.counts || !a.out_ids || !a.out_frames || !a.out_counts || !a.out_source)
    return fail(h, -1, "%s: a required pointer is NULL", what);
  if (!a.token_logp != !a.out_token_logp || !a.path_logp != !a.out_path_logp)
    return fail(h, -1, "%s: token_logp / path_logp and their outputs go together", what);
  if (a.frame_logp && a.frame_pitch < a.T)
    return fail(h, -1, "%s: frame_pitch=%lld is less than T=%d", what, (long long)a.frame_pitch, a.T);
  int rows = 0, smem = 0;
  if (ctc_spot_plan(c.num_classes, &rows, &smem) == 1)
    return fail(h, -1, "%s: a frame of %d classes does not fit in shared memory", what, c.num_classes);
  const int64_t need = gam_ctc_bias_workspace_bytes(h, a.B, a.T, a.K, a.max_det);
  if (need < 0) return fail(h, -1, "%s: K=%d x max_det=%d candidates are too many", what, a.K, a.max_det);
  int32_t* ws = reinterpret_cast<int32_t*>(workspace_base(h, what, workspace, workspace_bytes, need, false));
  if (!ws) return -1;
  a.V1 = c.num_classes;
  a.log_theta = static_cast<float>(std::log(static_cast<double>(threshold)));   // spot's rounding
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int stage = 0; stage < 3; ++stage) {
    PROF(PC_ALIGN);
    launch_ctc_bias(a, ws, stage, s);
  }
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

int gam_ctc_bias(gam_handle* h, const float* log_probs, const int32_t* enc_len, int32_t B, int32_t T, const int32_t* keywords,
                 const int32_t* keyword_len, int32_t K, int32_t Umax, const int32_t* det_start, const int32_t* det_end,
                 const float* det_score, const int32_t* det_count, int32_t max_det, float threshold, const uint8_t* token_flags,
                 int32_t V, const int32_t* ids, const int32_t* frames, const int32_t* counts, int32_t max_out, const float* token_logp,
                 const float* path_logp, double* frame_logp, int64_t frame_pitch, void* workspace, int64_t workspace_bytes,
                 int32_t* out_ids, int32_t* out_frames, int32_t* out_counts, int32_t* out_source, float* out_token_logp,
                 float* out_path_logp, void* stream) {
  BiasArgs a{log_probs, enc_len, keywords, keyword_len, det_start, det_end, det_score, det_count, token_flags, ids, frames, counts,
             token_logp, path_logp, frame_logp, frame_pitch, B, T, 0, K, Umax, max_det, max_out, 0.f, out_ids, out_frames, out_counts,
             out_source, out_token_logp, out_path_logp};
  return ctc_bias_run(h, "ctc_bias", a, threshold, V, workspace, workspace_bytes, stream);
}

int64_t gam_ctc_bias_resume_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t K, int32_t max_det) {
  return gam_ctc_bias_workspace_bytes(h, B, T, K, max_det);
}

int gam_ctc_bias_resume(gam_handle* h, const float* log_probs, int32_t B, int32_t T, const int32_t* hi, const int32_t* frame_base,
                        const int32_t* finish, const int32_t* keywords, const int32_t* keyword_len, int32_t K, int32_t Umax,
                        const void* state, int64_t record_bytes, const int32_t* det_start, const int32_t* det_end,
                        const float* det_score, const int32_t* det_count, int32_t max_det, float threshold,
                        const uint8_t* token_flags, int32_t V, const int32_t* ids, const int32_t* frames, const int32_t* counts,
                        const int32_t* left_boundary, int32_t max_out, const float* token_logp, double* frame_logp,
                        int64_t frame_pitch, void* workspace, int64_t workspace_bytes, int32_t* out_ids, int32_t* out_frames,
                        int32_t* out_counts, int32_t* out_source, float* out_token_logp, int32_t* released_until,
                        int32_t* carry_start, int32_t* carry_end, float* carry_score, int32_t* carry_count, void* stream) {
  if (!hi || !frame_base || !finish || !left_boundary || !state || !released_until || !carry_start || !carry_end || !carry_score ||
      !carry_count)
    return fail(h, -1, "ctc_bias_resume: hi, frame_base, finish, left_boundary, state, released_until and carry_* are required");
  if (Umax >= 1 && Umax <= kSpotMaxTokens && record_bytes != ctc_spot_record_bytes(Umax))
    return fail(h, -1, "ctc_bias_resume: record_bytes=%lld, but Umax=%d needs %lld", (long long)record_bytes, Umax,
                (long long)ctc_spot_record_bytes(Umax));
  BiasArgs a{log_probs, hi, keywords, keyword_len, det_start, det_end, det_score, det_count, token_flags, ids, frames, counts,
             token_logp, nullptr, frame_logp, frame_pitch, B, T, 0, K, Umax, max_det, max_out, 0.f, out_ids, out_frames, out_counts,
             out_source, out_token_logp, nullptr, frame_base, finish, left_boundary, static_cast<const uint8_t*>(state), record_bytes,
             released_until, carry_start, carry_end, carry_score, carry_count};
  return ctc_bias_run(h, "ctc_bias_resume", a, threshold, V, workspace, workspace_bytes, stream);
}

int64_t gam_rnnt_align_scores_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || T <= 0 || T > h->max_t || U < 0 || U > kAlignMaxTokens) return -1;
  return gam_rnnt_joint_workspace_bytes(h, B, T, U + 1);
}

int gam_rnnt_align_scores(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, int32_t B, int32_t T, int32_t U,
                          void* workspace, int64_t workspace_bytes, float* blank, float* label, void* stream) {
  const gam_config& c = h->cfg;
  if (align_args(h, "rnnt_align_scores", 2, B, T, U) != 0) return -1;
  const int U1 = U + 1;
  if (joint_args(h, "rnnt_align_scores", B, T, U1, true) != 0) return -1;
  if (!enc || !dec || (U > 0 && !targets) || !blank || !label) return fail(h, -1, "rnnt_align_scores: a required pointer is NULL");
  uint8_t* ws = workspace_base(h, "rnnt_align_scores", workspace, workspace_bytes, gam_rnnt_align_scores_workspace_bytes(h, B, T, U),
                               true);
  if (!ws) return -1;
  ProjWs w;
  proj_layout(c, B, T, U1, ws, &w);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rnnt_project(h, enc, dec, B, T, U1, w.E, w.P, PC_RNNT_JOINT, s);
  int rc;
  { PROF(PC_RNNT_JOINT);
    rc = launch_rnnt_joint_gather(w.E, w.P, h->w.rnnt_wo, h->w.rnnt_bo, targets, blank, label, nullptr, B, T, U1, c.joint_hidden,
                                  c.num_classes, s); }
  if (rc != 0) return fail(h, -4, "rnnt_align_scores: launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "rnnt_align_scores");
  return 0;
}

int64_t gam_rnnt_align_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || T <= 0 || T > h->max_t || U < 0 || U > kAlignMaxTokens) return -1;
  return align_up(static_cast<int64_t>(B) * rnnt_bp_words(T, U) * 4, 1024);
}

int gam_rnnt_align(gam_handle* h, const float* blank, const float* label, const int32_t* enc_len, const int32_t* target_len, int32_t B,
                   int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, int32_t* frames, float* token_logp,
                   float* viterbi_logp, float* log_likelihood, int32_t* path_rows, void* stream) {
  if (align_args(h, "rnnt_align", 2, B, T, U) != 0) return -1;
  if (!blank || !label || !enc_len || !target_len || (U > 0 && (!frames || !token_logp)) || !viterbi_logp || !log_likelihood ||
      !path_rows)
    return fail(h, -1, "rnnt_align: a required pointer is NULL");
  uint8_t* ws = workspace_base(h, "rnnt_align", workspace, workspace_bytes, gam_rnnt_align_workspace_bytes(h, B, T, U), false);
  if (!ws) return -1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_ALIGN);   // one piece: the backpointers
    rc = launch_rnnt_align(blank, label, enc_len, target_len, B, T, U, reinterpret_cast<uint32_t*>(ws), frames, token_logp,
                           viterbi_logp, log_likelihood, path_rows, s); }
  if (rc != 0) return fail(h, -4, "rnnt_align: launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "rnnt_align");
  return 0;
}

// gam_rnnt_predict's U LSTM steps, one launch each.  Step u reads h from g[:, u-1] (steps are separate launches, so every block
// of step u sees all of step u-1).  c_seq == nullptr: the cell is updated in place in c1; otherwise step u's cell goes to
// c_seq[u] and the last one is copied to c1.
static int rnnt_predict_run(gam_handle* h, const char* what, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U,
                            float* g, float* h1, float* c1, float* c_seq, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 2) return fail(h, -1, "%s: model has no RNN-T head", what);
  if (B <= 0 || U <= 0) return fail(h, -1, "%s: bad sizes (B=%d, U=%d)", what, B, U);
  if (x == nullptr && U != 1) return fail(h, -1, "%s: without labels the step count U must be 1 (got %d)", what, U);
  if (c.pred_hidden > 1024) return fail(h, -1, "%s: pred_hidden %d exceeds 1024", what, c.pred_hidden);
  const int H = c.pred_hidden;
  const int64_t BH = static_cast<int64_t>(B) * H;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int u = 0; u < U; ++u) {
    const float* h_in = u == 0 ? h0 : g + static_cast<int64_t>(u - 1) * H;
    const int64_t pitch = u == 0 ? H : static_cast<int64_t>(U) * H;
    const float* c_in = u == 0 ? c0 : c_seq ? c_seq + (u - 1) * BH : c1;
    PROF(PC_RNNT_PREDICT);
    launch_lstm_step(x, U, u, c.num_classes, h->w.rnnt_emb_gates, h->w.rnnt_whh_t, h_in, pitch, c_in, g, u == U - 1 ? h1 : nullptr,
                     c_seq ? c_seq + u * BH : c1, B, H, s);
  }
  if (c_seq) cudaMemcpyAsync(c1, c_seq + (U - 1) * BH, BH * 4, cudaMemcpyDeviceToDevice, s);
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

int gam_rnnt_predict(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, float* g, float* h1,
                     float* c1, void* stream) {
  return rnnt_predict_run(h, "rnnt_predict", x, h0, c0, B, U, g, h1, c1, nullptr, stream);
}

int gam_rnnt_predict_train(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, float* g,
                           float* h1, float* c1, float* c_seq, void* stream) {
  return rnnt_predict_run(h, "rnnt_predict_train", x, h0, c0, B, U, g, h1, c1, c_seq, stream);
}

// ---- backward passes of the head calls (csrc/head_grads.cu)
int64_t gam_ctc_log_probs_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T) {
  if (!h || h->cfg.head != 1 || B <= 0 || T <= 0) return -1;
  CtcBwdWs w;
  return ctc_bwd_layout(h->cfg, static_cast<int64_t>(B) * T, nullptr, &w) + 1024;
}

int gam_ctc_log_probs_backward(gam_handle* h, const float* enc, int32_t B, int32_t T, const float* log_probs, const float* grad,
                               void* workspace, int64_t workspace_bytes, float* d_enc, float* dW, float* db, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 1) return fail(h, -1, "ctc_log_probs_backward: model has no CTC head");
  if (B <= 0 || T <= 0) return fail(h, -1, "ctc_log_probs_backward: bad sizes (B=%d, T=%d)", B, T);
  if ((dW == nullptr) != (db == nullptr)) return fail(h, -1, "ctc_log_probs_backward: dW and db go together");
  uint8_t* ws = workspace_base(h, "ctc_log_probs_backward", workspace, workspace_bytes,
                               gam_ctc_log_probs_backward_workspace_bytes(h, B, T), true);
  if (!ws) return -1;
  const int64_t R = static_cast<int64_t>(B) * T;
  CtcBwdWs w;
  ctc_bwd_layout(c, R, ws, &w);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_HEAD_BACKWARD);
    launch_softmax_grad(grad, log_probs, w.dl, R, c.num_classes, s); }
  if (dW != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_outer_sum(w.dl, enc, R, c.num_classes, c.d_model, dW, db, w.part, s); }
  if (d_enc != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_head_matmul(w.dl, h->w.ctc_w, c.d_model, 1, d_enc, R, c.num_classes, c.d_model, nullptr, nullptr, 1, 1, s); }
  GAM_CHECK_LAUNCH(h, "ctc_log_probs_backward");
  return 0;
}

int64_t gam_rnnt_joint_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || T <= 0 || U <= 0) return -1;
  JointBwdWs w;
  return joint_bwd_layout(h->cfg, B, T, U, nullptr, &w) + 1024;
}

int gam_rnnt_joint_backward(gam_handle* h, const float* enc, const float* dec, int32_t B, int32_t T, int32_t U, const float* log_probs,
                            const float* grad, void* workspace, int64_t workspace_bytes, float* d_enc, float* d_dec, float* dW_enc,
                            float* db_enc, float* dW_pred, float* db_pred, float* dW_out, float* db_out, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 2) return fail(h, -1, "rnnt_joint_backward: model has no RNN-T head");
  if (B <= 0 || T <= 0 || U <= 0) return fail(h, -1, "rnnt_joint_backward: bad sizes (B=%d, T=%d, U=%d)", B, T, U);
  if (joint_args(h, "rnnt_joint_backward", B, T, U, false) != 0) return -1;
  if ((dW_enc == nullptr) != (db_enc == nullptr) || (dW_pred == nullptr) != (db_pred == nullptr) || (dW_out == nullptr) != (db_out == nullptr))
    return fail(h, -1, "rnnt_joint_backward: each weight gradient goes with its bias gradient");
  uint8_t* ws = workspace_base(h, "rnnt_joint_backward", workspace, workspace_bytes, gam_rnnt_joint_backward_workspace_bytes(h, B, T, U),
                               true);
  if (!ws) return -1;
  JointBwdWs w;
  joint_bwd_layout(c, B, T, U, ws, &w);
  const int J = c.joint_hidden, V1 = c.num_classes;
  const int64_t BT = static_cast<int64_t>(B) * T, BU = static_cast<int64_t>(B) * U, rows = BT * U;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rnnt_project(h, enc, dec, B, T, U, w.E, w.P, PC_HEAD_BACKWARD, s);   // the forward's projections, the same bits
  { PROF(PC_HEAD_BACKWARD);
    launch_softmax_grad(grad, log_probs, w.dl, rows, V1, s); }
  if (dW_out != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_outer_sum_joint(w.dl, w.E, w.P, T, U, rows, V1, J, dW_out, db_out, w.part, s); }
  const bool need_hidden = d_enc || d_dec || dW_enc || dW_pred;
  if (need_hidden) {
    { PROF(PC_HEAD_BACKWARD);   // dhid = (dlogit W_o) * [hid > 0]
      launch_head_matmul(w.dl, h->w.rnnt_wo, J, 1, w.dhid, rows, V1, J, w.E, w.P, T, U, s); }
    { PROF(PC_HEAD_BACKWARD);   // dE[b, t] = sum_u dhid[b, t, u]
      launch_segment_sum(w.dhid, w.dE, BT, U, J, 1, U, 0, 1, s); }
    { PROF(PC_HEAD_BACKWARD);   // dP[b, u] = sum_t dhid[b, t, u]
      launch_segment_sum(w.dhid, w.dP, BU, T, J, U, static_cast<int64_t>(T) * U, 1, U, s); }
  }
  joint_input_grads(h, enc, dec, BT, BU, w.dE, w.dP, w.part, d_enc, d_dec, dW_enc, db_enc, dW_pred, db_pred, s);
  GAM_CHECK_LAUNCH(h, "rnnt_joint_backward");
  return 0;
}

int64_t gam_rnnt_predict_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t U) {
  if (!h || h->cfg.head != 2 || B <= 0 || U <= 0) return -1;
  PredBwdWs w;
  return pred_bwd_layout(h->cfg, B, U, nullptr, &w) + 1024;
}

int gam_rnnt_predict_backward(gam_handle* h, const int64_t* x, const float* h0, const float* c0, int32_t B, int32_t U, const float* g,
                              const float* c_seq, const float* grad_g, const float* grad_h1, const float* grad_c1, const float* embed,
                              const float* w_ih, const float* w_hh, void* workspace, int64_t workspace_bytes, float* d_h0, float* d_c0,
                              float* d_embed, float* dW_ih, float* dW_hh, float* d_bias, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 2) return fail(h, -1, "rnnt_predict_backward: model has no RNN-T head");
  if (B <= 0 || U <= 0) return fail(h, -1, "rnnt_predict_backward: bad sizes (B=%d, U=%d)", B, U);
  if (x == nullptr && U != 1) return fail(h, -1, "rnnt_predict_backward: without labels the step count U must be 1 (got %d)", U);
  const int H = c.pred_hidden, V1 = c.num_classes;
  if (H > lstm_bwd_max_hidden()) return fail(h, -1, "rnnt_predict_backward: pred_hidden %d exceeds %d", H, lstm_bwd_max_hidden());
  if (!g || !c_seq || !grad_g || !w_hh) return fail(h, -1, "rnnt_predict_backward: g, c_seq, grad_g and w_hh are required");
  if ((dW_hh == nullptr) != (d_bias == nullptr)) return fail(h, -1, "rnnt_predict_backward: dW_hh and d_bias go together");
  if ((dW_ih || d_embed) && (!embed || !w_ih)) return fail(h, -1, "rnnt_predict_backward: embed and w_ih are required for their grads");
  uint8_t* ws = workspace_base(h, "rnnt_predict_backward", workspace, workspace_bytes, gam_rnnt_predict_backward_workspace_bytes(h, B, U),
                               true);
  if (!ws) return -1;
  PredBwdWs w;
  pred_bwd_layout(c, B, U, ws, &w);
  const int64_t BH = static_cast<int64_t>(B) * H, BU = static_cast<int64_t>(B) * U;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (grad_c1 != nullptr)
    cudaMemcpyAsync(w.dcc, grad_c1, BH * 4, cudaMemcpyDeviceToDevice, s);
  else
    cudaMemsetAsync(w.dcc, 0, BH * 4, s);
  for (int u = U - 1; u >= -1; --u) {
    PROF(PC_HEAD_BACKWARD);
    launch_lstm_bwd_step(x, U, u, V1, h->w.rnnt_emb_gates, h->w.rnnt_whh_t, w_hh, h0, c0, g, c_seq, grad_g, grad_h1, w.dgates, w.dcc,
                         d_h0, d_c0, B, H, s);
  }
  if (dW_hh != nullptr) { PROF(PC_HEAD_BACKWARD);
    launch_outer_sum_shift(w.dgates, g, h0, U, BU, 4 * H, H, dW_hh, d_bias, w.part, s); }
  if (dW_ih != nullptr || d_embed != nullptr) {
    if (x == nullptr) {   // every step read the zero embedding
      if (dW_ih) cudaMemsetAsync(dW_ih, 0, static_cast<int64_t>(4) * H * H * 4, s);
      if (d_embed) cudaMemsetAsync(d_embed, 0, static_cast<int64_t>(V1) * H * 4, s);
    } else {
      { PROF(PC_HEAD_BACKWARD);
        if (launch_class_gate_sum(x, BU, w.dgates, 4 * H, V1, V1 - 1, w.dcls, s) != 0)
          return fail(h, -1, "rnnt_predict_backward: pred_hidden %d too large for the class sums", H); }
      if (dW_ih != nullptr) { PROF(PC_HEAD_BACKWARD);
        launch_outer_sum(w.dcls, embed, V1, 4 * H, H, dW_ih, nullptr, w.part, s); }
      if (d_embed != nullptr) { PROF(PC_HEAD_BACKWARD);
        launch_head_matmul(w.dcls, w_ih, H, 1, d_embed, V1, 4 * H, H, nullptr, nullptr, 1, 1, s); }
    }
  }
  GAM_CHECK_LAUNCH(h, "rnnt_predict_backward");
  return 0;
}

// ---- fused RNN-T loss (csrc/rnnt_loss.cu; stage 1 is the gathered joint of heads.cu with the row lse kept)
int64_t gam_rnnt_loss_saved_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!loss_sizes_ok(h, B, T, U)) return -1;
  return static_cast<int64_t>(3) * B * T * (U + 1) * 4;
}

int64_t gam_rnnt_loss_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!loss_sizes_ok(h, B, T, U)) return -1;
  LossFwdWs w;
  return loss_fwd_layout(h->cfg, B, T, U, nullptr, &w) + 1024;
}

int gam_rnnt_loss(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, const int32_t* enc_len,
                  const int32_t* target_len, int32_t B, int32_t T, int32_t U, void* workspace, int64_t workspace_bytes, float* saved,
                  float* loss, void* stream) {
  const gam_config& c = h->cfg;
  if (loss_args(h, "rnnt_loss", B, T, U) != 0) return -1;
  if (!enc || !dec || (U > 0 && !targets) || !enc_len || !target_len || !saved || !loss)
    return fail(h, -1, "rnnt_loss: a required pointer is NULL");
  uint8_t* ws = workspace_base(h, "rnnt_loss", workspace, workspace_bytes, gam_rnnt_loss_workspace_bytes(h, B, T, U), true);
  if (!ws) return -1;
  LossFwdWs w;
  loss_fwd_layout(c, B, T, U, ws, &w);
  const int J = c.joint_hidden, U1 = U + 1;
  const int64_t N = static_cast<int64_t>(B) * T * U1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rnnt_project(h, enc, dec, B, T, U1, w.E, w.P, PC_RNNT_JOINT, s);
  int rc;
  { PROF(PC_RNNT_JOINT);
    rc = launch_rnnt_joint_gather(w.E, w.P, h->w.rnnt_wo, h->w.rnnt_bo, targets, w.blank, w.label, saved, B, T, U1, J, c.num_classes, s); }
  if (rc != 0) return fail(h, -4, "rnnt_loss: stage 1 launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  { PROF(PC_ALIGN);
    launch_rnnt_loss_alpha_beta(w.blank, w.label, enc_len, target_len, B, T, U, w.alpha, saved + N, saved + 2 * N, loss, s); }
  GAM_CHECK_LAUNCH(h, "rnnt_loss");
  return 0;
}

int64_t gam_rnnt_loss_backward_workspace_bytes(const gam_handle* h, int32_t B, int32_t T, int32_t U) {
  if (!loss_sizes_ok(h, B, T, U)) return -1;
  LossBwdWs w;
  return loss_bwd_layout(h->cfg, B, T, U, nullptr, &w) + 1024;
}

int gam_rnnt_loss_backward(gam_handle* h, const float* enc, const float* dec, const int32_t* targets, const int32_t* enc_len,
                           const int32_t* target_len, int32_t B, int32_t T, int32_t U, const float* saved, const float* grad_loss,
                           void* workspace, int64_t workspace_bytes, float* d_enc, float* d_dec, float* dW_enc, float* db_enc,
                           float* dW_pred, float* db_pred, float* dW_out, float* db_out, void* stream) {
  const gam_config& c = h->cfg;
  if (loss_args(h, "rnnt_loss_backward", B, T, U) != 0) return -1;
  if (!enc || !dec || (U > 0 && !targets) || !enc_len || !target_len || !saved || !grad_loss)
    return fail(h, -1, "rnnt_loss_backward: a required pointer is NULL");
  if ((dW_enc == nullptr) != (db_enc == nullptr) || (dW_pred == nullptr) != (db_pred == nullptr) || (dW_out == nullptr) != (db_out == nullptr))
    return fail(h, -1, "rnnt_loss_backward: each weight gradient goes with its bias gradient");
  uint8_t* ws = workspace_base(h, "rnnt_loss_backward", workspace, workspace_bytes, gam_rnnt_loss_backward_workspace_bytes(h, B, T, U),
                               true);
  if (!ws) return -1;
  LossBwdWs w;
  loss_bwd_layout(c, B, T, U, ws, &w);
  const int J = c.joint_hidden, V1 = c.num_classes, U1 = U + 1;
  const int64_t BT = static_cast<int64_t>(B) * T, BU1 = static_cast<int64_t>(B) * U1, N = BT * U1;
  const RnntLossPlan plan = rnnt_loss_plan(B, T, U, V1);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rnnt_project(h, enc, dec, B, T, U1, w.E, w.P, PC_HEAD_BACKWARD, s);   // the forward's projections, the same bits
  const bool need_hidden = d_enc || d_dec || dW_enc || dW_pred;
  if (need_hidden || dW_out) {
    const RnntLossArgs a{w.E, w.P, h->w.rnnt_wo, h->w.rnnt_bo, targets, enc_len, target_len, saved, saved + N, saved + 2 * N, grad_loss,
                         B, T, U, J, V1};
    int rc;
    { PROF(PC_HEAD_BACKWARD);
      rc = launch_rnnt_loss_grads(a, plan, need_hidden ? w.dE_part : nullptr, w.dP_part, w.part, dW_out, db_out, s); }
    if (rc != 0) return fail(h, -4, "rnnt_loss_backward: launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  }
  if (need_hidden) {
    { PROF(PC_HEAD_BACKWARD);   // dE[b, t] = sum over the column strips, in strip order
      launch_segment_sum(w.dE_part, w.dE, BT, plan.NS, J, 1, 1, 0, BT, s); }
    { PROF(PC_HEAD_BACKWARD);   // dP[b, u] = sum over the frame ranges, in range order
      launch_segment_sum(w.dP_part, w.dP, BU1, plan.ST, J, 1, 1, 0, BU1, s); }
  }
  joint_input_grads(h, enc, dec, BT, BU1, w.dE, w.dP, w.part, d_enc, d_dec, dW_enc, db_enc, dW_pred, db_pred, s);
  GAM_CHECK_LAUNCH(h, "rnnt_loss_backward");
  return 0;
}

int64_t gam_emo_workspace_bytes(const gam_handle* h, int32_t B, int32_t T) {
  if (!h || h->cfg.head != 3 || B < 1 || T < 1 || T > 65535 * kPoolChunk) return -1;
  return static_cast<int64_t>(B) * pool_chunk_count(T) * h->cfg.d_model * 4;
}

int gam_emo_head(gam_handle* h, const float* enc, const int32_t* enc_len, int32_t B, int32_t T, void* workspace,
                 int64_t workspace_bytes, float* pooled, float* logits, float* probs, void* stream) {
  const gam_config& c = h->cfg;
  if (c.head != 3) return fail(h, -1, "emo_head: model has no emo head");
  if (B < 1 || T < 1 || T > 65535 * kPoolChunk)
    return fail(h, -1, "emo_head: bad sizes (B=%d, T=%d; 1 <= T <= %d)", B, T, 65535 * kPoolChunk);
  float* part = reinterpret_cast<float*>(workspace_base(h, "emo_head", workspace, workspace_bytes, gam_emo_workspace_bytes(h, B, T),
                                                        false));   // one piece: the per-chunk sums
  if (!part) return -1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_EMO_HEAD);
    launch_pool_chunks(enc, enc_len, B, T, part, s); }
  { PROF(PC_EMO_HEAD);
    launch_pooled_head(part, enc_len, B, T, h->w.emo_w, h->w.emo_b, c.num_classes, pooled, logits, probs, s); }
  GAM_CHECK_LAUNCH(h, "emo_head");
  return 0;
}

int gam_emo_frame_logits(gam_handle* h, const float* enc, int32_t B, int32_t T, const int32_t* lo, const int32_t* hi, const int32_t* dst,
                         float* frame_logits, int32_t n_frames, void* stream) {
  if (!h) return -1;
  if (h->cfg.head != 3) return fail(h, -1, "emo_frame_logits: model has no emo head");
  if (B < 1 || B > 65535) return fail(h, -1, "emo_frame_logits: B=%d outside [1, 65535]", B);
  if (T < 1 || n_frames < 1) return fail(h, -1, "emo_frame_logits: bad sizes (T=%d, n_frames=%d; both must be >= 1)", T, n_frames);
  if (!enc || !lo || !hi || !dst || !frame_logits) return fail(h, -1, "emo_frame_logits: NULL pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_EMO_FRAME_LOGITS);
    launch_emo_frame_logits(enc, B, T, lo, hi, dst, h->w.emo_w, h->w.emo_b, h->cfg.num_classes, frame_logits, n_frames, s); }
  GAM_CHECK_LAUNCH(h, "emo_frame_logits");
  return 0;
}

int gam_emo_spans(gam_handle* h, const float* frame_logits, int32_t n_frames, const int32_t* span_start, const int32_t* span_end,
                  int32_t S, float* logits, float* probs, void* stream) {
  if (!h) return -1;
  if (h->cfg.head != 3) return fail(h, -1, "emo_spans: model has no emo head");
  if (n_frames < 1 || S < 1) return fail(h, -1, "emo_spans: bad sizes (n_frames=%d, S=%d; both must be >= 1)", n_frames, S);
  if (!frame_logits || !span_start || !span_end) return fail(h, -1, "emo_spans: NULL pointer");
  if (!logits && !probs) return 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_EMO_SPANS);
    launch_emo_spans(frame_logits, n_frames, h->cfg.num_classes, span_start, span_end, S, logits, probs, s); }
  GAM_CHECK_LAUNCH(h, "emo_spans");
  return 0;
}

int gam_group_words(gam_handle* h, const int32_t* ids, const int32_t* frames, const int32_t* counts, int32_t B, int32_t max_out,
                    const uint8_t* token_flags, int32_t V, int32_t max_words, int32_t* word_start, int32_t* word_end,
                    int32_t* word_first_token, int32_t* word_tokens, int32_t* n_words, void* stream) {
  if (B < 0 || max_out <= 0 || max_words <= 0 || V <= 0) return fail(h, -1, "group_words: bad sizes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_MISC);
    launch_group_words(ids, frames, counts, token_flags, B, V, max_out, max_words, word_start, word_end, word_first_token, word_tokens,
                       n_words, s); }
  GAM_CHECK_LAUNCH(h, "group_words");
  return 0;
}

int gam_resample(gam_handle* h, const float* x, int64_t x_pitch, int32_t B, const int64_t* spans, const float* table,
                 int32_t table_rows, int32_t table_cols, int32_t o, int32_t n, float* y, int64_t y_pitch, void* stream) {
  if (!h) return -1;
  if (!x || !spans || !table || !y) return fail(h, -1, "resample: NULL pointer");
  if (B < 1 || B > 65535) return fail(h, -1, "resample: B=%d outside [1, 65535]", B);
  if (x_pitch < 0 || y_pitch < 0 || (y_pitch + 255) / 256 > INT32_MAX)
    return fail(h, -1, "resample: bad row pitch (x %lld, y %lld)", (long long)x_pitch, (long long)y_pitch);
  // w: torchaudio's ceil(lowpass_filter_width * orig / (min(orig, new) * rolloff)), in the same double operations
  const int32_t w = (o < 1 || n < 1) ? -1 : static_cast<int32_t>(std::ceil(6.0 * o / (std::min(o, n) * 0.99)));
  const int32_t taps = table_rows;
  if (w < 0 || table_cols != n || taps != 2 * static_cast<int64_t>(w) + o || static_cast<int64_t>(taps) * n > (int64_t(1) << 20))
    return fail(h, -1, "resample: a table of %d x %d does not match o=%d, n=%d (2 w + o = %lld taps x n phases, w = %d, at most 2^20 "
                "entries)", table_rows, table_cols, o, n, 2 * static_cast<long long>(w) + o, n, w);
  if (y_pitch == 0) return 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_MISC);
    launch_resample(x, x_pitch, table, n, o, w, taps, spans, B, y, y_pitch, s); }
  GAM_CHECK_LAUNCH(h, "resample");
  return 0;
}

int gam_comm_unique_id(uint8_t* out128) { return comm_unique_id(out128); }

int gam_comm_init(gam_handle* h, const uint8_t* id128, int32_t rank, int32_t nranks) {
  if (nranks < 1 || rank < 0 || rank >= nranks) return fail(h, -1, "comm_init: bad rank %d of %d", rank, nranks);
  if (h->comm) { comm_destroy(h->comm); h->comm = nullptr; }
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, -11, "cudaSetDevice(%d) failed", h->device);
  const char* err = "";
  const int rc = comm_init(&h->comm, id128, rank, nranks, &err);
  if (rc != 0) return fail(h, -20, "NCCL communicator init failed (rank %d of %d): %s", rank, nranks, err);
  h->comm_rank = rank;
  h->comm_nranks = nranks;
  return 0;
}

int32_t gam_comm_nccl_version(void) { return comm_nccl_version(); }

int gam_gather_hyps(gam_handle* h, const int32_t* packed, int64_t n_int32, int32_t* gathered, void* stream) {
  if (!h->comm) return fail(h, -20, "gather_hyps: no communicator (call gam_comm_init first)");
  if (n_int32 <= 0) return fail(h, -1, "gather_hyps: empty payload");
  const char* err = "";
  { cudaStream_t s = static_cast<cudaStream_t>(stream);
    PROF(PC_MISC);
    if (comm_all_gather_i32(h->comm, packed, gathered, n_int32, s, &err) != 0) return fail(h, -20, "ncclAllGather failed: %s", err); }
  return 0;
}

int gam_profile_begin(gam_handle* h) {
  for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
  h->prof_ev.clear();
  h->prof_cls.clear();
  h->prof = true;
  return 0;
}

int gam_profile_end(gam_handle* h, double* ms_per_class, int64_t* launches_per_class, int32_t n_classes) {
  h->prof = false;
  for (int i = 0; i < n_classes; ++i) { ms_per_class[i] = 0.0; launches_per_class[i] = 0; }
  int rc = 0;
  for (size_t i = 0; i < h->prof_cls.size(); ++i) {
    float ms = 0.f;
    if (cudaEventSynchronize(h->prof_ev[2 * i + 1]) != cudaSuccess ||
        cudaEventElapsedTime(&ms, h->prof_ev[2 * i], h->prof_ev[2 * i + 1]) != cudaSuccess) { rc = -1; continue; }
    const int cls = h->prof_cls[i];
    if (cls < n_classes) { ms_per_class[cls] += ms; launches_per_class[cls] += 1; }
  }
  for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
  h->prof_ev.clear();
  h->prof_cls.clear();
  if (rc) return fail(h, -5, "profile: an event could not be read: %s", cudaGetErrorString(cudaGetLastError()));
  return 0;
}

int gam_profile_class_count(void) { return PC_COUNT; }

const char* gam_profile_class_name(int32_t cls) {
  static const char* names[PC_COUNT] = {"logmel", "subsample_conv1", "gemm_conv2_implicit", "gemm_subsample_out", "gemm_ffn_up_silu",
                                        "gemm_ffn_down_res", "gemm_qkv", "gemm_proj_res", "gemm_pw1_glu", "layernorm", "attention",
                                        "dwconv_bn_silu", "ctc_head_argmax", "ctc_collapse", "rnnt_enc_proj", "rnnt_greedy", "misc",
                                        "ctc_log_probs", "rnnt_joint", "rnnt_predict", "emo_head", "head_backward", "align", "emo_frame_logits",
                                        "emo_spans"};
  return (cls >= 0 && cls < PC_COUNT) ? names[cls] : "?";
}

int gam_test_gemm(gam_handle* h, int32_t kind, const void* A, const void* A2, int32_t n1, const void* W, const float* bias,
                  const float* res, void* out, int32_t M, int32_t N, int32_t K, int32_t ldo, int32_t col0, float scale,
                  int32_t reverse, const int32_t* m_dev, void* stream) {
  if (kind < GEMM_BIAS_F16 || (kind > GEMM_BIAS_F32 && kind != kTestGemmPower))
    return fail(h, -1, "test_gemm: unknown kind %d", kind);
  if (!A || !W || !out || (kind != kTestGemmPower && !bias) || (kind == GEMM_BIAS_RES_F32 && !res))
    return fail(h, -1, "test_gemm: A, W, out, bias (and res for kind 3) are required");
  if (M <= 0 || N <= 0 || N % 256 != 0 || K <= 0 || K % 64 != 0) return fail(h, -1, "test_gemm: bad sizes M=%d N=%d K=%d", M, N, K);
  // GLU and power write one column per pair of accumulator columns; f32 epilogues store float2, f16 ones half2
  const int ncol = (kind == GEMM_BIAS_GLU_F16 || kind == kTestGemmPower) ? N / 2 : N;
  if (col0 < 0 || col0 % 2 != 0 || ldo % 2 != 0 || ldo < col0 + ncol)
    return fail(h, -1, "test_gemm: columns [%d, %d) do not fit an even row pitch %d", col0, col0 + ncol, ldo);
  if (A2 && (kind != GEMM_BIAS_F16 || n1 <= 0 || n1 >= N || n1 % 256 != 0))
    return fail(h, -1, "test_gemm: a second A operand needs kind 0 and 0 < n1 < N, n1 %% 256 == 0 (n1=%d)", n1);
  CUtensorMap ta, ta2, tw;
  int rc = make_tmap_2d_f16(&ta, A, M, K, K, 128, 64);
  if (A2) rc |= make_tmap_2d_f16(&ta2, A2, M, K, K, 128, 64);
  rc |= make_tmap_2d_f16(&tw, W, N, K, K, 128, 64);
  if (rc) return fail(h, -2, "tensor map encode failed (rc=%d)", rc);
  const size_t esz = (kind == GEMM_BIAS_RES_F32 || kind == GEMM_BIAS_F32 || kind == kTestGemmPower) ? 4 : 2;
  void* o = static_cast<char*>(out) + col0 * esz;
  const float* r = res ? reinterpret_cast<const float*>(reinterpret_cast<const char*>(res) + col0 * esz) : nullptr;
  // output map of the shared-memory store path; a column range TMA cannot address is stored directly
  CUtensorMap to;
  const bool has_to = kind != kTestGemmPower && kind != GEMM_BIAS_RES_F32 && make_tmap_out(&to, o, esz == 4, M, ncol, ldo) == 0;
  h->test_gemm_slots = has_to ? 1 : 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    PROF(PC_MISC);
    if (kind == kTestGemmPower)
      rc = launch_gemm_power(&ta, &tw, M, N, K, static_cast<float*>(o), ldo, h->gemm_clusters, s);
    else if (A2)
      rc = launch_gemm_dual_a(&ta, &ta2, n1, &tw, M, N, K, bias, o, ldo, h->gemm_clusters, s, reverse, m_dev, has_to ? &to : nullptr);
    else
      rc = launch_gemm(kind, &ta, &tw, M, N, K, bias, r, o, ldo, scale, h->gemm_clusters, s, reverse, m_dev, has_to ? &to : nullptr);
  }
  if (rc) return fail(h, -4, "gemm launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "test_gemm");
  return 0;
}

int gam_test_gemm_used_slots(gam_handle* h) { return h->test_gemm_slots; }

int gam_test_gemm_conv(gam_handle* h, int32_t conv1d, const void* A, const void* W, const float* bias, const int32_t* len_out,
                       const int32_t* cu, const int32_t* plen, void* out, int32_t out_frames, int32_t B, int32_t T_in, int32_t F1,
                       int32_t C, int32_t taps, int32_t N, int32_t f32_out, void* stream) {
  if (!A || !W || !bias || !len_out || !out) return fail(h, -1, "test_gemm_conv: A, W, bias, len_out and out are required");
  if ((cu != nullptr) != (plen != nullptr)) return fail(h, -1, "test_gemm_conv: cu and plen go together");
  if (B <= 0 || T_in <= 0 || C <= 0 || C % 64 != 0 || N <= 0 || N % 256 != 0)
    return fail(h, -1, "test_gemm_conv: bad sizes B=%d T_in=%d C=%d N=%d (C %% 64 == 0, N %% 256 == 0)", B, T_in, C, N);
  if (!conv1d && F1 != 32)
    return fail(h, -1, "test_gemm_conv: the 3x3 conv maps 16 output bins per frame (F1 = 32), got F1=%d", F1);
  if (!conv1d && (taps != 9 || f32_out)) return fail(h, -1, "test_gemm_conv: the 3x3 conv has 9 taps and fp16 output");
  if (conv1d && (taps < 1 || taps % 2 == 0)) return fail(h, -1, "test_gemm_conv: conv1d needs an odd tap count (got %d)", taps);
  const int k = conv1d ? taps : 3;
  const int T_out = sub_out_len(T_in, k, (k - 1) / 2);
  if (T_out <= 0) return fail(h, -1, "test_gemm_conv: T_in=%d gives no output frame", T_in);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cu) {
    std::vector<int> c, p;
    if (dev_ints(cu, B, c, s) || dev_ints(plen, B, p, s)) return fail(h, -3, "test_gemm_conv: cannot read cu / plen");
    for (int b = 0; b < B; ++b)
      if (c[b] < 0 || static_cast<int64_t>(c[b]) + std::min(std::max(p[b], 0), T_out) > out_frames)
        return fail(h, -1, "test_gemm_conv: utterance %d (cu %d, plen %d) runs past %d output frames", b, c[b], p[b], out_frames);
  } else if (static_cast<int64_t>(B) * T_out > out_frames) {
    return fail(h, -1, "test_gemm_conv: %d x %d output frames do not fit %d", B, T_out, out_frames);
  }
  CUtensorMap ta, tw;
  int rc = conv1d ? make_tmap_conv3d(&ta, A, B, T_in, C) : make_tmap_conv4d(&ta, A, B, T_in, F1, C);
  rc |= make_tmap_2d_f16(&tw, W, N, static_cast<uint64_t>(taps) * C, static_cast<uint64_t>(taps) * C, 128, 64);
  if (rc) return fail(h, -2, "tensor map encode failed (rc=%d)", rc);
  {
    PROF(PC_MISC);
    rc = conv1d ? launch_gemm_conv1d(&ta, &tw, B, T_out, C, taps, N, bias, len_out, cu, plen, out, N, f32_out, h->gemm_clusters, s)
                : launch_gemm_conv(&ta, &tw, B, T_out, C, N, bias, len_out, cu, plen, out, N, h->gemm_clusters, s);
  }
  if (rc) return fail(h, -4, "conv gemm launch rejected (rc=%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, "test_gemm_conv");
  return 0;
}

int gam_test_layernorm(gam_handle* h, const float* x, const float* g, const float* b, void* out, int32_t rows, const int32_t* rows_dev,
                       int32_t reverse, void* stream) {
  if (!x || !g || !b || !out || rows <= 0) return fail(h, -1, "test_layernorm: x, g, b, out and rows > 0 are required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_LAYERNORM);
    launch_ln_f16(x, g, b, static_cast<__half*>(out), rows, rows_dev, reverse, s); }
  GAM_CHECK_LAUNCH(h, "test_layernorm");
  return 0;
}

int gam_test_ln_rope(gam_handle* h, const float* x, const float* g, const float* b, const float* rope_cos, const float* rope_sin,
                     int32_t table_rows, int32_t half_dim, void* out_u, void* out_r, int32_t rows, const int32_t* rows_dev,
                     const int32_t* row_t, int32_t T, int32_t reverse, void* stream) {
  if (!x || !g || !b || !rope_cos || !rope_sin || !out_u || !out_r || rows <= 0)
    return fail(h, -1, "test_ln_rope: every buffer and rows > 0 are required");
  if (half_dim <= 0 || half_dim % 4 != 0 || 768 % (2 * half_dim) != 0)
    return fail(h, -1, "test_ln_rope: half_dim %d must be a multiple of 4 and 2*half_dim divide 768", half_dim);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (row_t) {
    std::vector<int> n, t;
    int live = rows;
    if (rows_dev) {
      if (dev_ints(rows_dev, 1, n, s)) return fail(h, -3, "test_ln_rope: cannot read rows_dev");
      live = std::min(std::max(n[0], 0), rows);
    }
    if (live > 0 && dev_ints(row_t, live, t, s)) return fail(h, -3, "test_ln_rope: cannot read row_t");
    for (int r = 0; r < live; ++r)
      if (t[r] < 0 || t[r] >= table_rows) return fail(h, -1, "test_ln_rope: row %d has position %d outside the %d-row table", r, t[r], table_rows);
  } else if (T <= 0 || T > table_rows) {
    return fail(h, -1, "test_ln_rope: T=%d must be in [1, %d] without row_t", T, table_rows);
  }
  { PROF(PC_LAYERNORM);
    launch_ln_rope_f16(x, g, b, rope_cos, rope_sin, static_cast<__half*>(out_u), static_cast<__half*>(out_r), rows, rows_dev, row_t,
                       T > 0 ? T : 1, half_dim, reverse, s); }
  GAM_CHECK_LAUNCH(h, "test_ln_rope");
  return 0;
}

int gam_test_ln_out_ln(gam_handle* h, const float* r, const float* g_out, const float* b_out, const float* g_next, const float* b_next,
                       float* x_out, void* y_out, int32_t rows, const int32_t* rows_dev, int32_t reverse, void* stream) {
  if (!r || !g_out || !b_out || !x_out || rows <= 0 || (y_out && (!g_next || !b_next)))
    return fail(h, -1, "test_ln_out_ln: r, g_out, b_out, x_out, rows > 0 (and g_next, b_next with y_out) are required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_LAYERNORM);
    launch_ln_out_ln(r, g_out, b_out, g_next, b_next, x_out, static_cast<__half*>(y_out), rows, rows_dev, reverse, s); }
  GAM_CHECK_LAUNCH(h, "test_ln_out_ln");
  return 0;
}

int gam_test_unpack_rows(gam_handle* h, const float* x, const float* gamma, const float* beta, const int32_t* cu, const int32_t* plen,
                         float* out, int32_t B, int32_t T, int32_t rows, int32_t reverse, void* stream) {
  if (!x || !cu || !plen || !out || (gamma != nullptr) != (beta != nullptr) || B <= 0 || T <= 0)
    return fail(h, -1, "test_unpack_rows: x, cu, plen, out, B > 0, T > 0 (and gamma with beta) are required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<int> c, p;
  if (dev_ints(cu, B, c, s) || dev_ints(plen, B, p, s)) return fail(h, -3, "test_unpack_rows: cannot read cu / plen");
  for (int b = 0; b < B; ++b) {
    const int n = std::min(p[b], T);
    if (n > 0 && (c[b] < 0 || static_cast<int64_t>(c[b]) + n > rows))
      return fail(h, -1, "test_unpack_rows: utterance %d (cu %d, plen %d) reads past %d rows", b, c[b], p[b], rows);
  }
  { PROF(PC_MISC);
    launch_unpack_rows(x, gamma, beta, cu, plen, out, B, T, reverse, s); }
  GAM_CHECK_LAUNCH(h, "test_unpack_rows");
  return 0;
}

int gam_test_dwconv(gam_handle* h, int32_t layer_norm, const void* g, const float* w, const float* bias, const float* gamma,
                    const float* beta, const int32_t* len, const int32_t* cu, const int32_t* plen, const int32_t* row_b,
                    const int32_t* row_t, const int32_t* rows_dev, void* out, int32_t B, int32_t T, int32_t rows, int32_t kw,
                    void* stream) {
  if (!g || !w || !bias || !len || !out || B <= 0 || T <= 0) return fail(h, -1, "test_dwconv: g, w, bias, len, out, B, T are required");
  if (kw != 5 && kw != 31) return fail(h, -1, "test_dwconv: kernel size %d (5 or 31 are compiled)", kw);
  if ((cu != nullptr) != (plen != nullptr)) return fail(h, -1, "test_dwconv: cu and plen go together");
  if (layer_norm && (!gamma || !beta || (cu && (!row_b || !row_t))))
    return fail(h, -1, "test_dwconv: the LayerNorm variant needs gamma, beta (and row_b, row_t when packed)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<int> l, c, p;
  if (dev_ints(len, B, l, s)) return fail(h, -3, "test_dwconv: cannot read len");
  if (cu && (dev_ints(cu, B, c, s) || dev_ints(plen, B, p, s))) return fail(h, -3, "test_dwconv: cannot read cu / plen");
  for (int b = 0; b < B; ++b) {
    // rows of utterance b the kernel touches: reads frames < min(len, T), writes frames < min(plen, T) (padded: T)
    const int n = std::max(std::min(l[b], T), cu ? std::min(p[b], T) : T);
    const int64_t base = cu ? c[b] : static_cast<int64_t>(b) * T;
    if (n > 0 && (base < 0 || base + n > rows))
      return fail(h, -1, "test_dwconv: utterance %d (rows %lld + %d) runs past %d rows", b, (long long)base, n, rows);
  }
  if (layer_norm) {   // one warp per row < live rows; a packed row finds its (utterance, frame) in row_b / row_t
    int live = B * T;
    std::vector<int> n, rb, rt;
    if (rows_dev) {
      if (dev_ints(rows_dev, 1, n, s)) return fail(h, -3, "test_dwconv: cannot read rows_dev");
      live = std::min(std::max(n[0], 0), B * T);
    }
    if (live > rows) return fail(h, -1, "test_dwconv: %d live rows exceed the %d-row buffers", live, rows);
    if (cu && live > 0) {
      if (dev_ints(row_b, live, rb, s) || dev_ints(row_t, live, rt, s)) return fail(h, -3, "test_dwconv: cannot read row_b / row_t");
      for (int r = 0; r < live; ++r)
        if (rb[r] < 0 || rb[r] >= B || rt[r] < 0 || rt[r] >= T)
          return fail(h, -1, "test_dwconv: row %d maps to (utterance %d, frame %d) outside [%d, %d)", r, rb[r], rt[r], B, T);
    }
  }
  int rc;
  { PROF(PC_DWCONV);
    rc = layer_norm ? launch_dwconv_ln_silu(static_cast<const __half*>(g), w, bias, gamma, beta, len, cu, row_b, row_t, rows_dev,
                                            static_cast<__half*>(out), B, T, kw, s)
                    : launch_dwconv_bn_silu(static_cast<const __half*>(g), w, bias, len, cu, plen, static_cast<__half*>(out), B, T, kw, s); }
  if (rc) return fail(h, -4, "test_dwconv: launch rejected (kw=%d)", kw);
  GAM_CHECK_LAUNCH(h, "test_dwconv");
  return 0;
}

int gam_test_pack_plan(gam_handle* h, const int64_t* mel_len, int32_t B, int32_t k, int64_t M, int32_t* len0, int32_t* len1,
                       int32_t* len2, int32_t* plen, int32_t* run1, int32_t* cu, int32_t* rows_dev, int32_t* row_b, int32_t* row_t,
                       void* stream) {
  if (!mel_len || !len0 || !len1 || !len2 || !plen || !run1 || !cu || !rows_dev || !row_b || !row_t)
    return fail(h, -1, "test_pack_plan: every buffer is required");
  if (B <= 0 || B > 65535 || k < 1 || M <= 0 || M > INT32_MAX) return fail(h, -1, "test_pack_plan: bad sizes B=%d k=%d M=%lld", B, k, (long long)M);
  const int pad = (k - 1) / 2;
  const int T1 = sub_out_len(static_cast<int>(M), k, pad), T2 = sub_out_len(T1, k, pad);
  if (T2 <= 0) return fail(h, -1, "test_pack_plan: M=%lld gives no encoder frame", (long long)M);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_MISC);
    launch_pack_plan(reinterpret_cast<const long long*>(mel_len), B, 2 * pad - k, static_cast<int>(M), T1, T2, len0, len1, len2, plen,
                     run1, cu, rows_dev, row_b, row_t, s); }
  GAM_CHECK_LAUNCH(h, "test_pack_plan");
  return 0;
}

int gam_test_subsample_conv1(gam_handle* h, const float* mel, const int32_t* len0, const int32_t* len1, const int32_t* run1,
                             const float* w, const float* bias, void* out, int32_t B, int32_t F, int64_t M, int32_t C, void* stream) {
  if (!mel || !len0 || !len1 || !w || !bias || !out || B <= 0 || M <= 0 || M > INT32_MAX)
    return fail(h, -1, "test_subsample_conv1: mel, len0, len1, w, bias, out, B > 0, M > 0 are required");
  if (F <= 0 || F > 70 || C <= 0 || C % 8 != 0 || C / 8 > 128)
    return fail(h, -1, "test_subsample_conv1: F=%d (<= 70) or C=%d (multiple of 8, <= 1024) unsupported", F, C);
  const int T1 = sub_out_len(static_cast<int>(M), 3, 1), F1 = sub_out_len(F, 3, 1);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_SUB_CONV1);
    rc = launch_subsample_conv1(mel, len0, len1, run1, w, bias, static_cast<__half*>(out), B, static_cast<int>(M), F, T1, F1, C, s); }
  if (rc) return fail(h, -4, "test_subsample_conv1: launch rejected");
  GAM_CHECK_LAUNCH(h, "test_subsample_conv1");
  return 0;
}

int gam_test_mel_to_tmajor(gam_handle* h, const float* mel, const int32_t* len0, void* out, int32_t B, int32_t F, int64_t M, void* stream) {
  if (!mel || !len0 || !out || B <= 0 || B > 65535 || F <= 0 || M <= 0 || M > INT32_MAX)
    return fail(h, -1, "test_mel_to_tmajor: mel, len0, out and sizes B in [1, 65535], F > 0, M > 0 are required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  { PROF(PC_SUB_CONV1);
    launch_mel_to_tmajor_f16(mel, len0, static_cast<__half*>(out), B, F, static_cast<int>(M), s); }
  GAM_CHECK_LAUNCH(h, "test_mel_to_tmajor");
  return 0;
}

int gam_test_frames_split(gam_handle* h, const float* wav, int32_t B, int64_t n_samples, void* A, int32_t* fexp, void* stream) {
  const gam_config& c = h->cfg;
  if (!wav || !A || !fexp || B <= 0 || B > 65535 || n_samples > INT32_MAX)
    return fail(h, -1, "test_frames_split: wav, A, fexp and B in [1, 65535] are required");
  const int64_t M = gam_logmel_frames(h, n_samples);
  if (M <= 0) return fail(h, -1, "waveform too short: %lld samples", (long long)n_samples);
  if (c.center && n_samples <= c.n_fft / 2) return fail(h, -1, "reflect padding needs more than n_fft/2 samples");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_LOGMEL);
    rc = launch_frames_split(wav, B, static_cast<int>(n_samples), static_cast<int>(M), h->w.window, static_cast<__half*>(A), fexp,
                             c.n_fft, logmel_kp(c), c.hop_length, c.center, s); }
  if (rc) return fail(h, -4, "test_frames_split: launch rejected (n_fft %d)", c.n_fft);
  GAM_CHECK_LAUNCH(h, "test_frames_split");
  return 0;
}

int gam_test_mel_log(gam_handle* h, const float* P, const int32_t* fexp, int32_t B, int32_t M, int32_t nbins, const float* fb,
                     const int32_t* mel_lo, const int32_t* mel_hi, int32_t n_mels, float* mel, void* stream) {
  if (!P || !fexp || !fb || !mel_lo || !mel_hi || !mel || B <= 0 || B > 65535 || M <= 0)
    return fail(h, -1, "test_mel_log: P, fexp, fb, mel_lo, mel_hi, mel and B in [1, 65535], M > 0 are required");
  if (nbins <= 0 || nbins > 256 || n_mels <= 0 || n_mels > 64)
    return fail(h, -1, "test_mel_log: nbins %d (<= 256) or n_mels %d (<= 64) unsupported", nbins, n_mels);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<int> lo, hi;
  if (dev_ints(mel_lo, n_mels, lo, s) || dev_ints(mel_hi, n_mels, hi, s)) return fail(h, -3, "test_mel_log: cannot read mel_lo / mel_hi");
  for (int m = 0; m < n_mels; ++m)
    if (lo[m] < 0 || hi[m] > nbins) return fail(h, -1, "test_mel_log: mel %d bin range [%d, %d) outside [0, %d)", m, lo[m], hi[m], nbins);
  int rc;
  { PROF(PC_LOGMEL);
    rc = launch_mel_log(P, fexp, 256, B, M, nbins, fb, mel_lo, mel_hi, mel, n_mels, s); }
  if (rc) return fail(h, -4, "test_mel_log: launch rejected");
  GAM_CHECK_LAUNCH(h, "test_mel_log");
  return 0;
}

static int test_rnnt_greedy(gam_handle* h, const char* what, const float* encproj, const int32_t* len, const float* emb_gates,
                            const float* whhT, const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T,
                            int32_t V1, int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts,
                            float* token_logp, float* path_logp, int32_t* path_rows, int32_t* plan, void* stream,
                            const BoostGraph* boost = nullptr) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  { PROF(PC_RNNT_GREEDY);
    rc = launch_rnnt_greedy(encproj, emb_gates, whhT, wpT, bp, wo, bo, B, T, 320, V1, V1 - 1, max_symbols,
                            fresh_io(len, ids, frames, counts, max_out, token_logp, path_logp, path_rows), boost, plan, s); }
  if (rc > 0) return fail(h, -1, "%s: 16-CTA clusters cannot be scheduled on this device", what);
  if (rc < 0) return fail(h, -4, "%s: launch failed: %s", what, cudaGetErrorString(cudaGetLastError()));
  GAM_CHECK_LAUNCH(h, what);
  return 0;
}

int gam_test_rnnt_greedy_scored(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                                const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                                int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts,
                                float* token_logp, float* path_logp, int32_t* path_rows, int32_t* plan, void* stream) {
  if (!encproj || !len || !emb_gates || !whhT || !wpT || !bp || !wo || !bo || !ids || !frames || !counts || !token_logp || !path_logp ||
      !path_rows)
    return fail(h, -1, "test_rnnt_greedy_scored: every operand is required");
  if (B <= 0 || T <= 0 || V1 < 2 || max_symbols <= 0 || max_out <= 0)
    return fail(h, -1, "test_rnnt_greedy_scored: bad sizes (B=%d, T=%d, V1=%d, max_symbols=%d, max_out=%d)", B, T, V1, max_symbols,
                max_out);
  return test_rnnt_greedy(h, "test_rnnt_greedy_scored", encproj, len, emb_gates, whhT, wpT, bp, wo, bo, B, T, V1, max_symbols, max_out,
                          ids, frames, counts, token_logp, path_logp, path_rows, plan, stream);
}

int gam_test_rnnt_greedy_boost(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                               const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                               int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts, float* token_logp,
                               float* path_logp, int32_t* path_rows, const int32_t* boost_next, const float* boost_bonus,
                               int32_t n_states, int32_t* plan, void* stream) {
  if (!encproj || !len || !emb_gates || !whhT || !wpT || !bp || !wo || !bo || !ids || !frames || !counts ||
      (token_logp && (!path_logp || !path_rows)))
    return fail(h, -1, "test_rnnt_greedy_boost: every operand is required (path_logp and path_rows when token_logp is given)");
  if (B <= 0 || T <= 0 || V1 < 2 || max_symbols <= 0 || max_out <= 0)
    return fail(h, -1, "test_rnnt_greedy_boost: bad sizes (B=%d, T=%d, V1=%d, max_symbols=%d, max_out=%d)", B, T, V1, max_symbols,
                max_out);
  BoostGraph g;
  if (!boost_args(h, "test_rnnt_greedy_boost", boost_next, boost_bonus, n_states, &g)) return -1;
  return test_rnnt_greedy(h, "test_rnnt_greedy_boost", encproj, len, emb_gates, whhT, wpT, bp, wo, bo, B, T, V1, max_symbols, max_out,
                          ids, frames, counts, token_logp, path_logp, path_rows, plan, stream, &g);
}

int gam_test_rnnt_greedy(gam_handle* h, const float* encproj, const int32_t* len, const float* emb_gates, const float* whhT,
                         const float* wpT, const float* bp, const float* wo, const float* bo, int32_t B, int32_t T, int32_t V1,
                         int32_t max_symbols, int32_t max_out, int32_t* ids, int32_t* frames, int32_t* counts, int32_t* plan,
                         void* stream) {
  if (!encproj || !len || !emb_gates || !whhT || !wpT || !bp || !wo || !bo || !ids || !frames || !counts)
    return fail(h, -1, "test_rnnt_greedy: every operand is required");
  if (B <= 0 || T <= 0 || V1 < 2 || max_symbols <= 0 || max_out <= 0)
    return fail(h, -1, "test_rnnt_greedy: bad sizes (B=%d, T=%d, V1=%d, max_symbols=%d, max_out=%d)", B, T, V1, max_symbols, max_out);
  return test_rnnt_greedy(h, "test_rnnt_greedy", encproj, len, emb_gates, whhT, wpT, bp, wo, bo, B, T, V1, max_symbols, max_out, ids,
                          frames, counts, nullptr, nullptr, nullptr, plan, stream);
}

int gam_test_attention(gam_handle* h, const void* qkv, const int32_t* klen, void* out, int32_t B, int32_t T, void* stream) {
  const gam_config& c = h->cfg;
  if (T > h->max_t) return fail(h, -1, "test_attention: T=%d exceeds the handle's %d-frame limit", T, h->max_t);
  CUtensorMap tq;
  const uint64_t d = c.d_model;
  int rc = make_tmap_2d_f16(&tq, qkv, static_cast<uint64_t>(B) * T, 3 * d, 3 * d, 128, 64);
  if (rc) return fail(h, -2, "tensor map encode failed (rc=%d)", rc);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    PROF(PC_ATTENTION);
    rc = launch_attention(&tq, klen, nullptr, static_cast<__half*>(out), B, T, c.n_heads, c.d_model / c.n_heads, c.d_model, s);
  }
  if (rc) return fail(h, -4, "attention launch rejected (T=%d)", T);
  GAM_CHECK_LAUNCH(h, "test_attention");
  return 0;
}

int gam_test_attention_relpos(gam_handle* h, const void* qkv, const void* pos, const int32_t* klen, void* out, int32_t B,
                              int32_t T, void* stream) {
  const gam_config& c = h->cfg;
  if (T > h->max_t) return fail(h, -1, "test_attention_relpos: T=%d exceeds the handle's %d-frame limit", T, h->max_t);
  CUtensorMap tq, tp;
  const uint64_t d = c.d_model;
  int rc = make_tmap_2d_f16(&tq, qkv, static_cast<uint64_t>(B) * T, 4 * d, 4 * d, 128, 64);
  rc |= make_tmap_2d_f16(&tp, pos, 2 * static_cast<uint64_t>(h->max_t) - 1, d, d, 128, 64);
  if (rc) return fail(h, -2, "tensor map encode failed (rc=%d)", rc);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    PROF(PC_ATTENTION);
    rc = launch_attention_relpos(&tq, &tp, h->max_t, klen, nullptr, static_cast<__half*>(out), B, T, c.n_heads, c.d_model / c.n_heads,
                                 c.d_model, s);
  }
  if (rc) return fail(h, -4, "rel_pos attention launch rejected (T=%d, rc=%d)", T, rc);
  GAM_CHECK_LAUNCH(h, "test_attention_relpos");
  return 0;
}

int gam_test_attention_varlen(gam_handle* h, const void* qkv, const void* pos, const int32_t* klen, const int32_t* cu, void* out,
                              int32_t B, int32_t T, int32_t rows, void* stream) {
  const gam_config& c = h->cfg;
  if (!klen || !cu || rows <= 0) return fail(h, -1, "attention_varlen: klen, cu and rows are required");
  if (T > h->max_t) return fail(h, -1, "attention_varlen: T=%d exceeds the handle's %d-frame limit", T, h->max_t);
  CUtensorMap tq, tp;
  const uint64_t d = c.d_model, parts = pos ? 4 : 3;
  int rc = make_tmap_2d_f16(&tq, qkv, static_cast<uint64_t>(rows), parts * d, parts * d, 128, 64);
  if (pos) rc |= make_tmap_2d_f16(&tp, pos, 2 * static_cast<uint64_t>(h->max_t) - 1, d, d, 128, 64);
  if (rc) return fail(h, -2, "tensor map encode failed (rc=%d)", rc);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    PROF(PC_ATTENTION);
    rc = pos ? launch_attention_relpos(&tq, &tp, h->max_t, klen, cu, static_cast<__half*>(out), B, T, c.n_heads, c.d_model / c.n_heads,
                                       c.d_model, s)
             : launch_attention(&tq, klen, cu, static_cast<__half*>(out), B, T, c.n_heads, c.d_model / c.n_heads, c.d_model, s);
  }
  if (rc) return fail(h, -4, "varlen attention launch rejected (T=%d, rc=%d)", T, rc);
  GAM_CHECK_LAUNCH(h, "test_attention_varlen");
  return 0;
}

}  // extern "C"
