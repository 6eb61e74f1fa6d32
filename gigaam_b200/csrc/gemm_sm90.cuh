// Warp-specialised wgmma GEMM for sm_90a:  D[M,N] = A[M,K] * W[N,K]^T  (+ fused epilogue)
//
// Persistent CTAs, one per SM and paired into clusters (below), walk 128 x 256 output tiles.  Warp 0 of the producer
// warpgroup streams 64-wide k-blocks of A (128 rows) and W (256 rows, two 128-row TMA boxes) into a 4-stage shared-memory
// ring; the two consumer warpgroups each own 64 rows of the tile and issue wgmma.m64n256k16 with both operands read from
// shared memory (K-major, SWIZZLE_128B, exactly as TMA wrote them).  A stage goes back to the producer as soon as the
// wgmma group that read it has retired (one group stays in flight), so the loads of the next tile run under this tile's
// epilogue.
//
// Accumulators stay in registers (128 fp32 per consumer thread): the epilogue applies bias / residual / activation
// straight from the wgmma fragment (a thread holds two adjacent columns of two rows per 8-column block; four threads
// cover 32 contiguous bytes of a row, so every access fills whole 32-byte sectors).
//
// How a finished tile leaves the SM (A_2D epilogues but the residual and the DFT power): a tile whose 128 rows all lie
// below the live row count goes out through shared memory.  Each consumer warpgroup owns two 8 KB slots of 64 rows x 128
// bytes (64 fp16 or 32 fp32 columns, laid out as a SWIZZLE_128B TMA box, so the fragment writes are free of bank
// conflicts) and stores its 64 rows chunk by chunk, alternating slots: the leader waits until the bulk store issued from
// the slot two chunks ago has read it (wait_group.read 1), the warpgroup writes the chunk, fences it to the async proxy
// and the leader issues the bulk store.  The warpgroup goes on to the next tile without waiting for the stores, so the
// HBM traffic of the epilogue runs under the next main loop instead of stalling the tensor cores.  The tile that straddles the live row count, the
// phantom / dead half of a pair and the conv modes store straight from the fragment: no row at or past the live count is
// ever written.  EPI_BIAS_RES_F32 stores directly too: its residual loads stay on the epilogue's critical path, and
// loaded one chunk at a time for the slots they made more round trips than the direct path's batches (measured slower on
// an H100, with and without an L2 prefetch of the residual; DESIGN.md §7).  Only the instantiations that use the slots reserve them
// (gemm_smem_bytes): the others keep the shared memory, and so the L1 share of the unified L1 / shared memory, they had
// without them.
//
// Clusters of two CTAs share the weight tile.  The persistent grid walks pairs of tiles, m-blocks 2i and 2i + 1 of one
// n-block; the CTA of cluster rank r computes m-block 2i + r and loads W rows 128 r .. 128 r + 127 of the n-block with a
// TMA multicast into the same stage of both CTAs.  Each CTA so fetches 16 KB of A and 16 KB of W per k-block instead of
// 16 + 32 KB: the L2 -> shared-memory feed, which all SMs share, carries a third less per FLOP.  A pair is skipped only
// when both its blocks are dead; the phantom second block of an odd block count (and a dead block whose partner is
// live) still loads (TMA zero-fills rows past the tensor) and still arrives on every barrier, but stores nothing.
//
// Barriers: full[s] (one local producer arrival + 48 KB, of which 16 KB come from the peer's multicast and may land
// before the local expect_tx), empty[s] (one arrival per consumer warpgroup of BOTH CTAs: a stage is reloaded only when
// neither CTA still reads it, because either producer's multicast writes it in both).  A cluster barrier follows the
// barrier init and ends the kernel, so no CTA exits while its peer can still write into its shared memory or arrive
// on its barriers.
#pragma once
#include "gemm_params.cuh"

namespace gam {

constexpr int kG2Cluster = 2;   // CTAs per cluster, along M
constexpr int kG2Threads = 384;
constexpr int kG2Stages = 4;
constexpr int kG2BN = 256;
constexpr int kG2ABytes = 128 * 64 * 2;       // 16 KB: 128 rows of A
constexpr int kG2BBytes = 256 * 64 * 2;       // 32 KB: 256 rows of W
constexpr int kG2StageBytes = kG2ABytes + kG2BBytes;
constexpr int kG2SlotBytes = 64 * 128;          // 8 KB store slot: 64 rows x 128 bytes
constexpr int kG2StoreBytes = 2 * 2 * kG2SlotBytes;   // two slots per consumer warpgroup
constexpr int kG2BarBytes = 256;

template <int EPI, int AMODE>
constexpr bool gemm_tma_store() {
  return AMODE == A_2D && EPI != EPI_POWER_F32 && EPI != EPI_BIAS_RES_F32;
}
// dynamic shared memory: stages | store slots (only where used) | barriers, + 1 KB to align the base to 1024 bytes.
// 230 656 B with the slots (of the 232 448 B opt-in), 197 888 B without
template <int EPI, int AMODE>
constexpr int gemm_smem_bytes() {
  return kG2Stages * kG2StageBytes + (gemm_tma_store<EPI, AMODE>() ? kG2StoreBytes : 0) + kG2BarBytes + 1024;
}

// output row of local row `lr` (0..127) of 128-row block m_blk: whether it exists (is stored) and whether it lies
// inside the utterance's valid length (conv modes: ReLU value, else 0)
struct GemmRow {
  long long row;
  bool valid;
  bool live;
};

template <int AMODE>
__device__ __forceinline__ GemmRow gemm_row(const GemmParams& p, int m_rows, int m_blk, int lr) {
  GemmRow g;
  if constexpr (AMODE == A_2D) {
    g.row = static_cast<long long>(m_blk) * 128 + lr;
    g.valid = g.row < m_rows;
    g.live = true;
  } else {
    constexpr int kFramesPerBlock = (AMODE == A_CONV) ? 8 : 128;
    const bool blk_ok = m_blk < p.conv_num_blocks;
    const int b = blk_ok ? m_blk / p.conv_tiles_per_utt : 0;
    // A_CONV: a 128-row block is 8 output time steps x 16 frequency bins; A_CONV1D: 128 consecutive output frames
    const int t = (m_blk % p.conv_tiles_per_utt) * kFramesPerBlock + (AMODE == A_CONV ? (lr >> 4) : lr);
    const bool packed = p.conv_cu != nullptr;
    const long long base = (packed ? static_cast<long long>(__ldg(p.conv_cu + b)) : static_cast<long long>(b) * p.conv_T2) + t;
    g.row = AMODE == A_CONV ? base * 16 + (lr & 15) : base;
    const int tv = packed ? min(__ldg(p.conv_plen + b), p.conv_T2) : p.conv_T2;
    g.valid = blk_ok && t < tv;
    g.live = blk_ok && t < __ldg(p.conv_len2 + b);
  }
  return g;
}

// The epilogue arithmetic of fragment block i (columns 8 i + cq, + 1 of the tile) of row half h, shared by both store paths.
// bias (+ scale * residual) (+ SiLU); res is read only by EPI_BIAS_RES_F32
template <int EPI>
__device__ __forceinline__ float2 bias_act_pair(const float (&acc)[128], const float* bsrc, int i, int h, int cq, const float2& res,
                                                float scale) {
  const float2 bv = __ldg(reinterpret_cast<const float2*>(bsrc + 8 * i + cq));
  float x0 = acc[4 * i + 2 * h] + bv.x, x1 = acc[4 * i + 2 * h + 1] + bv.y;
  if constexpr (EPI == EPI_BIAS_RES_F32) {
    x0 = fmaf(scale, x0, res.x);
    x1 = fmaf(scale, x1, res.y);
  }
  if constexpr (EPI == EPI_BIAS_SILU_F16) { x0 = silu_f(x0); x1 = silu_f(x1); }
  return make_float2(x0, x1);
}
// GLU, i < 16: value columns [0,128) of the tile, gate columns [128,256)
__device__ __forceinline__ uint32_t glu_pair(const float (&acc)[128], const float* bsrc, int i, int h, int cq) {
  const int c = 8 * i + cq;
  const float2 ba = __ldg(reinterpret_cast<const float2*>(bsrc + c));
  const float2 bb = __ldg(reinterpret_cast<const float2*>(bsrc + 128 + c));
  const float g0 = (acc[4 * i + 2 * h] + ba.x) * sigmoid_f(acc[4 * (i + 16) + 2 * h] + bb.x);
  const float g1 = (acc[4 * i + 2 * h + 1] + ba.y) * sigmoid_f(acc[4 * (i + 16) + 2 * h + 1] + bb.y);
  return pack_half2(g0, g1);
}

// One consumer warpgroup's 64 rows (row0 ..) of a tile whose rows are all live, out through the warpgroup's two store slots
// (see the header).  rw: the thread's first row inside the 64 (the second is rw + 8).  Each chunk is 64 rows x 128 bytes:
// 8 fragment blocks of fp16 or 4 of fp32.  The chunk count per tile is even, so chunk c always uses slot c & 1 and the slot
// written now is the one whose bulk store was committed two groups ago: wait_group.read 1 frees it.
template <int EPI>
__device__ __forceinline__ void store_tile_tma(const GemmParams& p, const CUtensorMap& tmap_out, const float (&acc)[128],
                                               uint8_t* slots, int row0, int n_blk, int rw, int cq, int wg, bool leader) {
  constexpr bool kF32 = EPI == EPI_BIAS_F32;
  constexpr int kChunkBlocks = kF32 ? 4 : 8;
  constexpr int kOutCols = EPI == EPI_BIAS_GLU_F16 ? kG2BN / 2 : kG2BN;
  constexpr int kChunks = kOutCols / (8 * kChunkBlocks);   // 8 (fp32), 4 (fp16) or 2 (GLU)
  static_assert(kChunks % 2 == 0, "chunk c must map to slot c & 1 in every tile");
  const float* bsrc = p.bias + n_blk * kG2BN;
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
    uint8_t* slot = slots + (c & 1) * kG2SlotBytes;
    if (leader) ptx::tma_store_wait_read<1>();
    ptx::named_bar_sync<128>(1 + wg);   // the slot is free for every thread of the warpgroup
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rw + 8 * h;
#pragma unroll
      for (int j = 0; j < kChunkBlocks; ++j) {
        const int i = c * kChunkBlocks + j;
        if constexpr (EPI == EPI_BIAS_GLU_F16) {
          *reinterpret_cast<uint32_t*>(slot + ptx::sw128_off(r, 8 * j + cq) + 2 * cq) = glu_pair(acc, bsrc, i, h, cq);
        } else {
          const float2 x = bias_act_pair<EPI>(acc, bsrc, i, h, cq, make_float2(0.f, 0.f), p.scale);
          if constexpr (kF32)
            *reinterpret_cast<float2*>(slot + ptx::sw128_off_f32(r, 8 * j + cq) + 4 * (cq & 3)) = x;
          else
            *reinterpret_cast<uint32_t*>(slot + ptx::sw128_off(r, 8 * j + cq) + 2 * cq) = pack_half2(x.x, x.y);
        }
      }
    }
    ptx::fence_proxy_async_smem();      // this thread's slot writes are visible to the bulk store ...
    ptx::named_bar_sync<128>(1 + wg);   // ... and so are every other thread's
    if (leader) {
      ptx::tma_store_2d(&tmap_out, slot, n_blk * kOutCols + c * 8 * kChunkBlocks, row0);
      ptx::tma_store_commit();
    }
  }
}

template <int EPI, int AMODE>
__global__ void __cluster_dims__(kG2Cluster, 1, 1) __launch_bounds__(kG2Threads, 1)
gemm_f16_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2,
                   const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_out,
                   const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kG2Stages * kG2ABytes;
  uint8_t* smem_store = smem + kG2Stages * kG2StageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_store + (gemm_tma_store<EPI, AMODE>() ? kG2StoreBytes : 0));
  uint64_t* empty_bar = full_bar + kG2Stages;

  const int warp_idx = threadIdx.x >> 5;
  // packed rows: the row count of an A_2D product may live on the device (GemmParams::m_dev); every role derives the same
  // tile list from it, and CTAs the host sized for the padded maximum simply find no tile
  int m_rows = p.M, num_m_tiles = p.num_m_tiles;          // num_m_tiles counts 128-row blocks
  if constexpr (AMODE == A_2D) {
    if (p.m_dev != nullptr) {
      m_rows = min(max(__ldg(p.m_dev), 0), p.M);
      num_m_tiles = (m_rows + 127) >> 7;
    }
  }
  // both CTAs of a cluster walk the same list of tile pairs; rank r takes m-block 2 * m_pair + r
  const int crank = static_cast<int>(ptx::cluster_ctarank());
  const int num_pairs = ((num_m_tiles + 1) >> 1) * p.num_n_tiles;
  const int cluster_id = blockIdx.x / kG2Cluster, num_clusters = gridDim.x / kG2Cluster;
  // conv modes with packed output: a 128-row block whose first frame lies past the utterance's length produces nothing;
  // a pair of two such blocks (or of one and the phantom block past the last) is skipped by every role of both CTAs
  // (same predicate, same pair list)
  [[maybe_unused]] auto conv_tile_dead = [&](int m_blk) -> bool {
    if constexpr (AMODE == A_2D) {
      return false;
    } else {
      if (p.conv_cu == nullptr) return false;
      if (m_blk >= num_m_tiles) return true;
      constexpr int kFramesPerBlock = (AMODE == A_CONV) ? 8 : 128;
      return (m_blk % p.conv_tiles_per_utt) * kFramesPerBlock >= __ldg(p.conv_plen + m_blk / p.conv_tiles_per_utt);
    }
  };
  auto pair_dead = [&](int m_pair) -> bool { return conv_tile_dead(2 * m_pair) && conv_tile_dead(2 * m_pair + 1); };
  // every row of the block is live: the tile leaves through the store slots (see the header)
  auto tma_tile = [&](int m_blk) -> bool {
    if constexpr (gemm_tma_store<EPI, AMODE>()) return p.tma_out != 0 && (m_blk + 1) * 128 <= m_rows;
    return false;
  };

  if (warp_idx == 0 && ptx::elect_one()) {
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_a2);
    ptx::prefetch_tmap(&tmap_w);
    if constexpr (gemm_tma_store<EPI, AMODE>()) {
      if (p.tma_out) ptx::prefetch_tmap(&tmap_out);
    }
    for (int s = 0; s < kG2Stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2 * kG2Cluster);   // one arrival per consumer warpgroup of every CTA in the cluster
    }
    ptx::fence_mbar_init();
  }
  __syncwarp();
  ptx::cluster_sync();   // the peer's barriers are initialised before the first multicast or remote arrival reaches them

  if (warp_idx < 4) {
    // ===================================================== TMA producer (warp 0 of warpgroup 0)
    ptx::setmaxnreg_dec<40>();
    if (warp_idx == 0 && ptx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int pr = cluster_id; pr < num_pairs; pr += num_clusters) {
        const int pl = p.reverse ? num_pairs - 1 - pr : pr;
        const int m_pair = pl / p.num_n_tiles;
        const int n_blk = pl % p.num_n_tiles;
        if (pair_dead(m_pair)) continue;
        const int m_blk = 2 * m_pair + crank;
        const CUtensorMap* ta = (p.a1_nblks > 0 && n_blk >= p.a1_nblks) ? &tmap_a2 : &tmap_a;
        [[maybe_unused]] int conv_b = 0, conv_t0 = 0;
        if constexpr (AMODE == A_CONV) {
          conv_b = m_blk / p.conv_tiles_per_utt;
          conv_t0 = (m_blk % p.conv_tiles_per_utt) * 8;
        }
        if constexpr (AMODE == A_CONV1D) {
          conv_b = m_blk / p.conv_tiles_per_utt;
          conv_t0 = (m_blk % p.conv_tiles_per_utt) * 128;
        }
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          ptx::mbar_arrive_expect_tx(&full_bar[stage], kG2StageBytes);
          uint8_t* sa = smem_a + stage * kG2ABytes;
          if constexpr (AMODE == A_2D) {
            ptx::tma_load_2d(sa, ta, &full_bar[stage], kb * kGemmBK, m_blk * 128);
          } else if constexpr (AMODE == A_CONV1D) {
            const int tap = kb / p.conv_kchunks;
            const int c0 = (kb % p.conv_kchunks) * kGemmBK;
            // 128 output frames t0.. read input frames 2 t + tap - pad: box of 256 input frames traversed with stride 2
            ptx::tma_load_3d(sa, &tmap_a, &full_bar[stage], c0, 2 * conv_t0 + tap - p.conv_pad, conv_b);
          } else {
            const int tap = kb / p.conv_kchunks;
            const int c0 = (kb % p.conv_kchunks) * kGemmBK;
            const int kt = tap / 3, kf = tap % 3;
            ptx::tma_load_4d(sa, &tmap_a, &full_bar[stage], c0, kf - 1, 2 * conv_t0 + kt - 1, conv_b);
          }
          // this CTA's 128-row half of the W tile, into the same stage of both CTAs
          ptx::tma_load_2d_multicast(smem_b + stage * kG2BBytes + crank * (kG2BBytes / kG2Cluster), &tmap_w, &full_bar[stage],
                                     kb * kGemmBK, n_blk * kG2BN + crank * (kG2BN / kG2Cluster), (1u << kG2Cluster) - 1);
          if (++stage == kG2Stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================================================== consumer warpgroups 1, 2: rows 64 (wg - 1) .. + 63 of the tile
    ptx::setmaxnreg_inc<232>();
    const int wg = (warp_idx >> 2) - 1;
    const int lane = threadIdx.x & 31;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int lr0 = wg * 64 + (warp_idx & 3) * 16 + (lane >> 2);   // local rows lr0, lr0 + 8
    const int cq = 2 * (lane & 3);                                 // column of d[4i] inside 8-column block i
    int stage = 0;
    uint32_t phase = 0;
    // a stage is released to the producers of both CTAs: either one's multicast writes it here
    auto release = [&](int s) {
      if (wg_leader)
        for (int c = 0; c < kG2Cluster; ++c) ptx::mbar_arrive_cluster(&empty_bar[s], c);
    };
    for (int pr = cluster_id; pr < num_pairs; pr += num_clusters) {
      const int pl = p.reverse ? num_pairs - 1 - pr : pr;
      const int m_pair = pl / p.num_n_tiles;
      const int n_blk = pl % p.num_n_tiles;
      if (pair_dead(m_pair)) continue;
      const int m_blk = 2 * m_pair + crank;

      float acc[128];
      int prev = -1;
      for (int kb = 0; kb < p.num_k_blocks; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = ptx::smem_u32(smem_a + stage * kG2ABytes + wg * (64 * 128));
        const uint32_t b_addr = ptx::smem_u32(smem_b + stage * kG2BBytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBK / 16; ++k)
          ptx::wgmma_m64n256k16_f16(acc, ptx::make_wgmma_desc_sw128(a_addr + k * 32), ptx::make_wgmma_desc_sw128(b_addr + k * 32),
                                    (kb | k) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();   // the group of the previous k-block has retired: its stage is free
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == kG2Stages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      // the accumulators are final only now: keep the compiler from reading them ahead of the wait
#pragma unroll
      for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(acc[i])::"memory");
      if (prev >= 0) release(prev);

      if constexpr (gemm_tma_store<EPI, AMODE>()) {
        if (tma_tile(m_blk)) {
          store_tile_tma<EPI>(p, tmap_out, acc, smem_store + wg * 2 * kG2SlotBytes, m_blk * 128 + wg * 64, n_blk,
                              (warp_idx & 3) * 16 + (lane >> 2), cq, wg, wg_leader);
          continue;
        }
      }
      // ---- epilogue straight from the fragment
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const GemmRow gr = gemm_row<AMODE>(p, m_rows, m_blk, lr0 + 8 * h);
        if (!gr.valid) continue;
        if constexpr (EPI == EPI_POWER_F32) {
          // |X|^2 of a DFT whose cos rows fill accumulator columns [0,128) of the tile and sin rows [128,256)
          float* outp = reinterpret_cast<float*>(p.out) + static_cast<size_t>(gr.row) * p.ldo + n_blk * 128;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float ra = acc[4 * i + 2 * h], rb = acc[4 * i + 2 * h + 1];
            const float ia = acc[4 * (i + 16) + 2 * h], ib = acc[4 * (i + 16) + 2 * h + 1];
            float2 o;
            o.x = (ra * ra + ia * ia) * p.scale;   // undo the operand pre-scaling
            o.y = (rb * rb + ib * ib) * p.scale;
            *reinterpret_cast<float2*>(outp + 8 * i + cq) = o;
          }
        } else if constexpr (EPI == EPI_BIAS_GLU_F16) {
          // value columns [0,128) of the tile, gate columns [128,256): output column n_blk * 128 + c
          const float* bsrc = p.bias + n_blk * kG2BN;
          __half* outp = reinterpret_cast<__half*>(p.out) + static_cast<size_t>(gr.row) * p.ldo + n_blk * 128;
#pragma unroll
          for (int i = 0; i < 16; ++i) *reinterpret_cast<uint32_t*>(outp + 8 * i + cq) = glu_pair(acc, bsrc, i, h, cq);
        } else {
          const float* bsrc = p.bias + n_blk * kG2BN;
          const size_t base = static_cast<size_t>(gr.row) * p.ldo + static_cast<size_t>(n_blk) * kG2BN;
          // residual loads go out 16 at a time, each batch before its first store: the output may alias the residual
          // (in place), so the compiler keeps a load that follows a store behind it, and one load per store made every
          // load of the row wait out a full memory latency of its own
          constexpr int kBatch = 16;
#pragma unroll
          for (int i0 = 0; i0 < 32; i0 += kBatch) {
            [[maybe_unused]] float2 res[kBatch];
            if constexpr (EPI == EPI_BIAS_RES_F32) {
#pragma unroll
              for (int j = 0; j < kBatch; ++j) res[j] = *reinterpret_cast<const float2*>(p.res + base + 8 * (i0 + j) + cq);
            }
#pragma unroll
            for (int i = i0; i < i0 + kBatch; ++i) {
              const int c = 8 * i + cq;
              const float2 x = bias_act_pair<EPI>(acc, bsrc, i, h, cq, res[i - i0], p.scale);
              float x0 = x.x, x1 = x.y;
              if constexpr (EPI == EPI_CONV_RELU_MASK_F16 || EPI == EPI_CONV_RELU_MASK_F32) {
                x0 = gr.live ? fmaxf(x0, 0.f) : 0.f;
                x1 = gr.live ? fmaxf(x1, 0.f) : 0.f;
              }
              if constexpr (EPI == EPI_BIAS_RES_F32 || EPI == EPI_BIAS_F32 || EPI == EPI_CONV_RELU_MASK_F32) {
                *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + base + c) = make_float2(x0, x1);
              } else {
                *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(p.out) + base + c) = pack_half2(x0, x1);
              }
            }
          }
        }
      }
    }
    // the slots are not reused any more, but the kernel ends only once its stores have landed
    if (gemm_tma_store<EPI, AMODE>() && wg_leader) ptx::tma_store_wait<0>();
  }
  __syncwarp();
  ptx::cluster_sync();   // the peer may still multicast into this CTA's stages and arrive on its barriers until here
}

}  // namespace gam
