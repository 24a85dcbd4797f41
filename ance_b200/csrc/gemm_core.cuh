// gemm_core.cuh — the wgmma mainloops of this repo: tc05_gemm_kernel (below) and tc05_gemm_wide_kernel (a 128 x 256
// tile on two MMA warpgroups for the encoder's large bias / residual layers; see its own comment further down).
//
//   D[M,N] = A[M,K] * B[N,K]^T        A, B: 16-bit (bf16 or fp16), K-major, fp32 accumulate
//
// Used by (i) the encoder's linear layers (x * W^T, W stored [out,in] as in the checkpoint) and
// (ii) the coarse pass of the flat inner-product search (Q * P^T).  The two differ only in the
// epilogue functor `Ep` (bias/GELU/residual store vs. per-query running top-k).
//
// Structure (one CTA per SM, persistent, warp-specialised):
//   warp 0     : TMA producer  — streams 128x64 A and BNx64 B tiles through a STAGES-deep smem ring
//   warps 4-7  : MMA warpgroup — wgmma m64nBNk16 (two per 16-wide K step: rows 0-63 and 64-127), fp32
//                accumulators in registers; at the end of a tile they are written to a shared-memory
//                accumulator tile (row-major fp32) and the warpgroup moves on to the next tile
//   warps 8+   : epilogue      — read the accumulator tile (thread = row), run Ep, release the tile
// The register accumulators and the shared tile form a two-deep pipeline: the epilogue of tile i runs
// under the mainloop of tile i + 1.
// CG = 2 pairs two CTAs (cluster 2x1x1) on one 256-row tile: each CTA computes its own 128 A rows,
// the BN B rows are shared — each CTA loads half of them and multicasts it into both CTAs' rings.
//
// A "work item" is (m_blk, split): one M tile swept over a contiguous range of N blocks.  Plain
// GEMMs use one N block per work item; the search sweeps thousands, carrying top-k state.
#pragma once
#include "tc05.cuh"

namespace gemm {

using namespace tc05;

constexpr int BM = 128;  // rows per CTA
constexpr int BK = 64;   // 64 x 16-bit = one 128-byte swizzle span
constexpr int MMA_K = 16;

struct WorkShape {
  int M, N, K;
  int num_m_blks;        // ceil(M / (BM*CG))
  int num_n_blks;        // ceil(N / BN)
  int n_splits;          // work items per m block
  int n_blks_per_split;  // ceil(num_n_blks / n_splits)
  unsigned long long hint_a, hint_b;  // L2 cache-policy words of the A / B tile loads (0 = the epilogue's default)
  // Soft barrier between CTA pairs that sweep the SAME B rows (search, n_splits == 1): pace[c] = progress of cluster c
  // in tiles; a producer does not run more than pace_window tiles ahead of the slowest cluster, so that a B tile fetched
  // from HBM by the first pair is still in L2 when the last pair asks for it.  null = off.
  int* pace;
  int pace_window;
  int pace_stride;   // clusters c, c + stride, c + 2 stride, ... sweep the same rows (1: all of them; n_splits: one wave of
                     // (query tile, row range) items, item w on cluster w, range = w % n_splits)
};

// Publish this cluster's progress and wait (bounded: ~100 us, then go on regardless — the barrier is a bandwidth
// optimisation, never a correctness requirement, and must not hang if the grid is not fully co-resident).
static __device__ __noinline__ void pace_wait(int* pace, int window, int me, int n_clusters, int stride, int seq) {
  volatile int* vp = pace;
  vp[me] = seq;
  const long long t0 = clock64();
  for (;;) {
    int mn = 0x7fffffff;
    for (int c = me % stride; c < n_clusters; c += stride) mn = min(mn, vp[c]);
    if (seq - mn <= window || clock64() - t0 > 200000ll) break;
  }
}

struct EpiCtx {
  int m_blk, split;
  int nb0, nb1;     // n-block range of this work item
  int row0;         // first global row of this CTA's 128-row tile
  int quad;         // 32-row quarter of the tile this warp reads (warp_idx % 4)
  int epi_warp;     // 0 .. EPI_WARPS-1
  int lane;
  int work_seq;     // how many work items this CTA has processed before this one
  uint8_t* ep_smem; // Ep::kSmemBytes of shared memory owned by the epilogue (1024-B aligned)
};

template <int BN, int STAGES, int CG, int EP_SMEM = 0>
struct SmemPlan {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;            // the whole B tile in every CTA of the cluster
  static constexpr int kBHalfRows = BN / CG;              // rows of it this CTA loads (and multicasts when CG = 2)
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = STAGES * kStageBytes;
  static constexpr int kAccPitch = BN + 4;                // fp32 words per accumulator row
  static constexpr int kAccOffset = kRingBytes;
  static constexpr int kAccBytes = (BM * kAccPitch * 4 + 1023) / 1024 * 1024;
  static constexpr int kEpOffset = kAccOffset + kAccBytes;
  static constexpr int kBarOffset = kEpOffset + EP_SMEM;
  // full[STAGES] empty[STAGES] acc_full acc_empty
  static constexpr int kBarBytes = (2 * STAGES + 2) * 8;
  static constexpr int kTotal = kBarOffset + kBarBytes;
  static constexpr int kDynamicBytes = kTotal + 1024;  // slack for manual 1024-B alignment
  static_assert(kDynamicBytes <= 232448, "GEMM shared memory exceeds 227 KB");
};

template <uint32_t FMT, int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (BN == 128) wgmma_n128<FMT, 0>(d, adesc, bdesc, accumulate);
  else wgmma_n64<FMT, 0>(d, adesc, bdesc, accumulate);
}

template <class Ep, int BN, int STAGES, int CG, int EPI_WARPS, uint32_t FMT>
__global__ void __launch_bounds__(256 + 32 * EPI_WARPS, 1)
tc05_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const WorkShape ws, const __grid_constant__ typename Ep::Params ep) {
  static_assert(BN == 64 || BN == 128, "BN");
  static_assert(CG == 1 || CG == 2, "CG");
  using Plan = SmemPlan<BN, STAGES, CG, Ep::kSmemBytes>;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* acc_tile = reinterpret_cast<float*>(smem + Plan::kAccOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Plan::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* afull_bar = empty_bar + STAGES;
  uint64_t* aempty_bar = afull_bar + 1;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = (CG == 2) ? cluster_ctarank() : 0u;
  const bool leader = (cta_rank == 0);
  const int cluster_id = (CG == 2) ? (blockIdx.x >> 1) : blockIdx.x;
  const int num_clusters = (CG == 2) ? (gridDim.x >> 1) : gridDim.x;
  const int total_work = ws.num_m_blks * ws.n_splits;
  const int num_kb = (ws.K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);        // this CTA's producer arrives once; A + both B halves complete on it
      mbar_init(&empty_bar[s], 4 * CG);  // every MMA warp of every CTA that multicasts into this stage
    }
    mbar_init(afull_bar, 4);
    mbar_init(aempty_bar, EPI_WARPS);
    fence_barrier_init();
  }
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();

  if (warp == 0) {
    // ===================================== TMA producer =====================================
    if (lane == 0) {
      const uint64_t hint_a = ws.hint_a ? ws.hint_a : Ep::kHintA, hint_b = ws.hint_b ? ws.hint_b : Ep::kHintB;
      Ring<STAGES> ring;
      for (int w = cluster_id; w < total_work; w += num_clusters) {
        const int m_blk = w / ws.n_splits, split = w - m_blk * ws.n_splits;
        const int nb0 = split * ws.n_blks_per_split;
        const int nb1 = min(nb0 + ws.n_blks_per_split, ws.num_n_blks);
        const int a_row = (m_blk * CG + (int)cta_rank) * BM;
        for (int nb = nb0; nb < nb1; ++nb) {
          if (ws.pace != nullptr && leader && ((nb - nb0) & 7) == 0)
            pace_wait(ws.pace, ws.pace_window, cluster_id, num_clusters, ws.pace_stride,
                      ((w - cluster_id) / num_clusters) * ws.num_n_blks + (nb - nb0));
          const int b_row = nb * BN + (int)cta_rank * Plan::kBHalfRows;
          for (int kb = 0; kb < num_kb; ++kb) {
            // CG = 2: the stage is free only when the MMA warps of BOTH CTAs have released it (each of them arrives
            // on the empty barrier of both), since this CTA's half of B lands in the peer's ring too.
            mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1, 1);
            uint8_t* sa = smem + ring.stage * Plan::kStageBytes;
            uint8_t* sb = sa + Plan::kABytes + cta_rank * (Plan::kBHalfRows * 128);
            mbar_arrive_expect_tx(&full_bar[ring.stage], Plan::kStageBytes);
            tma_load_2d(sa, &tmA, &full_bar[ring.stage], kb * BK, a_row, hint_a);
            if constexpr (CG == 1) tma_load_2d(sb, &tmB, &full_bar[ring.stage], kb * BK, b_row, hint_b);
            else tma_load_2d_multicast(sb, &tmB, &full_bar[ring.stage], kb * BK, b_row, 0x3, hint_b);
            ring.advance();
          }
        }
      }
      if (ws.pace != nullptr && leader) *reinterpret_cast<volatile int*>(ws.pace + cluster_id) = 0x7fffffff;   // done: never the slowest
    }
  } else if (warp >= 4 && warp < 8) {
    // ===================================== MMA warpgroup ====================================
    Ring<STAGES> ring;
    uint32_t acc_phase = 0;
    auto release = [&](int stage) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[stage]);
        if constexpr (CG == 2) mbar_arrive_cluster(&empty_bar[stage], cta_rank ^ 1u);
      }
    };
    for (int w = cluster_id; w < total_work; w += num_clusters) {
      const int m_blk = w / ws.n_splits, split = w - m_blk * ws.n_splits;
      const int nb0 = split * ws.n_blks_per_split;
      const int nb1 = min(nb0 + ws.n_blks_per_split, ws.num_n_blks);
      (void)m_blk;
      for (int nb = nb0; nb < nb1; ++nb) {
        float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
        int prev_stage = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[ring.stage], ring.phase, 3);
          const uint32_t sa = smem_u32(smem + ring.stage * Plan::kStageBytes);
          const uint32_t sb = sa + Plan::kABytes;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / MMA_K; ++k) {
            const uint64_t bdesc = make_desc_k_sw128(sb + k * MMA_K * 2);
            wgmma_tile<FMT, BN>(acc0, make_desc_k_sw128(sa + k * MMA_K * 2), bdesc, 1u);
            wgmma_tile<FMT, BN>(acc1, make_desc_k_sw128(sa + 64 * 128 + k * MMA_K * 2), bdesc, 1u);
          }
          wgmma_commit();
          // the previous k block's wgmmas have finished reading their stage once at most one group is in flight
          wgmma_wait<1>();
          wgmma_fence_regs(acc0);
          wgmma_fence_regs(acc1);
          if (prev_stage >= 0) release(prev_stage);
          prev_stage = ring.stage;
          ring.advance();
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        if (prev_stage >= 0) release(prev_stage);
        // hand the tile to the epilogue once it has finished reading the previous one
        mbar_wait(aempty_bar, acc_phase ^ 1, 2);
        acc_store_frag(acc_tile, Plan::kAccPitch, 0, 0, acc0);
        acc_store_frag(acc_tile, Plan::kAccPitch, 64, 0, acc1);
        __syncwarp();
        if (lane == 0) mbar_arrive(afull_bar);
        acc_phase ^= 1;
      }
    }
  } else if (warp >= 8) {
    // ======================================= epilogue =======================================
    Ep epi;
    EpiCtx cx;
    cx.quad = warp & 3;
    cx.epi_warp = warp - 8;
    cx.lane = lane;
    cx.work_seq = 0;
    cx.ep_smem = smem + Plan::kEpOffset;
    uint32_t acc_phase = 0;
    const uint32_t tacc = smem_u32(acc_tile) / 4u + static_cast<uint32_t>((cx.quad * 32 + lane) * Plan::kAccPitch);
    for (int w = cluster_id; w < total_work; w += num_clusters, ++cx.work_seq) {
      cx.m_blk = w / ws.n_splits;
      cx.split = w - cx.m_blk * ws.n_splits;
      cx.nb0 = cx.split * ws.n_blks_per_split;
      cx.nb1 = min(cx.nb0 + ws.n_blks_per_split, ws.num_n_blks);
      cx.row0 = (cx.m_blk * CG + (int)cta_rank) * BM;
      epi.begin_work(ep, ws, cx);
      for (int nb = cx.nb0; nb < cx.nb1; ++nb) {
        mbar_wait(afull_bar, acc_phase, 4);
        epi.tile(ep, ws, cx, tacc, nb);
        __syncwarp();
        if (lane == 0) mbar_arrive(aempty_bar);
        acc_phase ^= 1;
      }
      epi.end_work(ep, ws, cx);
    }
    epi.end_kernel(ep, cx);
  }

  // no CTA of a pair may exit while its peer can still multicast into it or arrive on its barriers
  if constexpr (CG == 2) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// 128 x 256 tiles on two cooperating MMA warpgroups, epilogue from registers.
//
//   warpgroup 0  : warp 0 = TMA producer (128x64 A + 256x64 B per 48 KB stage, 3 stages); warps 1 and 2 = stagers of
//                  the output buffer, one per MMA warpgroup; 40 registers per thread (setmaxnreg)
//   warpgroup 1+g: rows 64g .. 64g+63 x 256 columns, one wgmma m64n256k16 per 16-wide K step (SS form, both operands
//                  in the ring); 128 fp32 accumulators per thread, 232 registers per thread
// Both warpgroups read the same B slice and their own half of the A slice.  Per 256 tensor clocks the wgmmas read
// 20 KB of shared memory and TMA writes 12 KB into it (the 128x128 tile: 160 B per clock, this one 128).
//
// Epilogue: the warpgroup runs Ep::tile on its accumulators, reading the residual from and writing the 16-bit output
// into its 64-row half of a 128x256 staging buffer.  Stager g then issues the TMA stores of that half and, once they
// have read it, the residual load of the next tile, so the residual lands during the next mainloop.  Two mbarriers
// per half: ready[g] (stager -> warpgroup: the residual has landed, or the half is free) and out[g] (warpgroup ->
// stager: the outputs are in the half).  The tensor cores idle while the epilogue runs: it suits epilogues that are
// a few hundred instructions per thread (bias, residual), not the GELU.
// ------------------------------------------------------------------------------------------------
constexpr int kWideBN = 256;
constexpr int kWideStages = 3;

template <int EP_SMEM>
struct WideSmemPlan {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = kWideBN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = kWideStages * kStageBytes;
  static constexpr int kEpOffset = kRingBytes;
  static constexpr int kBarOffset = kEpOffset + EP_SMEM;
  // full[STAGES] empty[STAGES] ready[2] out[2]
  static constexpr int kBarBytes = (2 * kWideStages + 4) * 8;
  static constexpr int kTotal = kBarOffset + kBarBytes;
  static constexpr int kDynamicBytes = kTotal + 1024;  // slack for manual 1024-B alignment
  static_assert(kDynamicBytes <= 232448, "GEMM shared memory exceeds 227 KB");
};

template <class Ep, uint32_t FMT>
__global__ void __launch_bounds__(384, 1)
tc05_gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const WorkShape ws, const __grid_constant__ typename Ep::Params ep) {
  using Plan = WideSmemPlan<Ep::kSmemBytes>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Plan::kBarOffset);
  uint64_t* empty_bar = full_bar + kWideStages;
  uint64_t* ready_bar = empty_bar + kWideStages;
  uint64_t* out_bar = ready_bar + 2;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int total_work = ws.num_m_blks * ws.num_n_blks;
  const int num_kb = (ws.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kWideStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // every warp of both MMA warpgroups
    }
    for (int g = 0; g < 2; ++g) {
      mbar_init(&ready_bar[g], 1);
      mbar_init(&out_bar[g], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ===================================== TMA producer =====================================
      Ring<kWideStages> ring;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int m_blk = w / ws.num_n_blks, nb = w - m_blk * ws.num_n_blks;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1, 1);
          uint8_t* sa = smem + ring.stage * Plan::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[ring.stage], Plan::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[ring.stage], kb * BK, m_blk * BM, Ep::kHintA);
          tma_load_2d(sa + Plan::kABytes, &tmB, &full_bar[ring.stage], kb * BK, nb * kWideBN, Ep::kHintB);
          ring.advance();
        }
      }
    } else if ((warp == 1 || warp == 2) && lane == 0) {
      // ====================== stager of MMA warpgroup g's half of the output buffer ======================
      const int g = warp - 1;
      uint8_t* half = smem + Plan::kEpOffset + g * (Ep::kSmemBytes / 2);
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int m_blk = w / ws.num_n_blks, nb = w - m_blk * ws.num_n_blks;
        const int row0 = m_blk * BM + 64 * g, col0 = nb * kWideBN;
        Ep::fill(ep, ws, half, &ready_bar[g], row0, col0);
        mbar_wait(&out_bar[g], phase, 2);
        phase ^= 1;
        Ep::drain(ep, ws, half, row0, col0);
      }
      bulk_wait_all();
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================================== MMA warpgroup g ====================================
    const int g = wg - 1;
    uint8_t* half = smem + Plan::kEpOffset + g * (Ep::kSmemBytes / 2);
    Ring<kWideStages> ring;
    uint32_t phase = 0;
    auto release = [&](int stage) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
    };
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      const int m_blk = w / ws.num_n_blks, nb = w - m_blk * ws.num_n_blks;
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[ring.stage], ring.phase, 3);
        const uint32_t sa = smem_u32(smem + ring.stage * Plan::kStageBytes);
        const uint32_t sb = sa + Plan::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k)
          wgmma_n256<FMT, 0>(acc, make_desc_k_sw128(sa + g * 64 * 128 + k * MMA_K * 2),
                             make_desc_k_sw128(sb + k * MMA_K * 2), 1u);
        wgmma_commit();
        // the previous k block's wgmmas have finished reading their stage once at most one group is in flight
        wgmma_wait<1>();
        wgmma_fence_regs(acc);
        if (prev_stage >= 0) release(prev_stage);
        prev_stage = ring.stage;
        ring.advance();
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev_stage);
      mbar_wait(&ready_bar[g], phase, 4);
      phase ^= 1;
      Ep::tile(ep, ws, acc, half, nb * kWideBN);
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&out_bar[g]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host-side launch helpers
// ------------------------------------------------------------------------------------------------
constexpr int kMaxDevices = 64;

inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}

// SM count of the CURRENT device (cached per device ordinal: one process may drive several GPUs through the C ABI)
inline int sm_count() {
  static int n[kMaxDevices] = {};
  const int dev = current_device();
  if (!n[dev]) cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
  return n[dev];
}

template <class Ep, int BN, int STAGES, int CG, int EPI_WARPS, uint32_t FMT>
cudaError_t launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const WorkShape& ws,
                   const typename Ep::Params& ep, int max_ctas, cudaStream_t stream) {
  using Plan = SmemPlan<BN, STAGES, CG, Ep::kSmemBytes>;
  auto kern = tc05_gemm_kernel<Ep, BN, STAGES, CG, EPI_WARPS, FMT>;
  static bool configured[kMaxDevices] = {};   // the opt-in is per device, not per process
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Plan::kDynamicBytes);
    if (e != cudaSuccess) return e;
    configured[dev] = true;
  }
  const int total = ws.num_m_blks * ws.n_splits;
  int clusters = min(total, (max_ctas > 0 ? max_ctas : sm_count()) / CG);
  if (clusters < 1) clusters = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(clusters * CG);
  cfg.blockDim = dim3(256 + 32 * EPI_WARPS);
  cfg.dynamicSmemBytes = Plan::kDynamicBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CG;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, tmA, tmB, ws, ep);
}

// tc05_gemm_wide_kernel: tmA box {64, BM}, tmB box {64, kWideBN}, ws = make_shape(M, N, K, kWideBN, 1, 0)
template <class Ep, uint32_t FMT>
cudaError_t launch_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, const WorkShape& ws,
                        const typename Ep::Params& ep, int max_ctas, cudaStream_t stream) {
  using Plan = WideSmemPlan<Ep::kSmemBytes>;
  auto kern = tc05_gemm_wide_kernel<Ep, FMT>;
  static bool configured[kMaxDevices] = {};
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Plan::kDynamicBytes);
    if (e != cudaSuccess) return e;
    configured[dev] = true;
  }
  const int ctas = max(1, min(ws.num_m_blks * ws.num_n_blks, max_ctas > 0 ? max_ctas : sm_count()));
  kern<<<ctas, 384, Plan::kDynamicBytes, stream>>>(tmA, tmB, ws, ep);
  return cudaGetLastError();
}

inline WorkShape make_shape(int M, int N, int K, int BN, int CG, int n_splits /* <=0: one N block per item */) {
  WorkShape ws;
  ws.M = M;
  ws.N = N;
  ws.K = K;
  ws.num_m_blks = (M + BM * CG - 1) / (BM * CG);
  ws.num_n_blks = (N + BN - 1) / BN;
  if (n_splits <= 0 || n_splits > ws.num_n_blks) n_splits = ws.num_n_blks;
  ws.n_blks_per_split = (ws.num_n_blks + n_splits - 1) / n_splits;
  ws.n_splits = (ws.num_n_blks + ws.n_blks_per_split - 1) / ws.n_blks_per_split;
  ws.hint_a = ws.hint_b = 0;
  ws.pace = nullptr;
  ws.pace_window = 0;
  ws.pace_stride = 1;
  return ws;
}

}  // namespace gemm
