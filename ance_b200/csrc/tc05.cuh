// tc05.cuh — sm_90a device primitives used by every tensor-core kernel in this repo:
// mbarrier, TMA (cp.async.bulk.tensor, with cluster multicast), wgmma (warpgroup MMA with
// shared-memory operand descriptors) and the shared-memory accumulator tiles the epilogues read.
// Inline PTX only; no CUTLASS dependency.
//
// Bit layouts of the descriptors follow the PTX ISA "wgmma matrix descriptor" tables.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace tc05 {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// L2 cache-policy words accepted by cp.async.bulk.tensor ... .L2::cache_hint
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst  = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast   = 0x14F0000000000000ull;

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// arrive on the barrier at the same smem offset in CTA `cta` of the cluster.  Used to hand a consumed ring stage back to
// the producer of another CTA: the consumer's reads of the stage are wgmma reads that wgmma.wait_group has already
// retired, so the arrive needs no ordering beyond its default .release.cta semantics.  The .release.cluster form compiles
// to MEMBAR.ALL.GPU + CCTL.IVALL, which the MMA warps would pay on every K block (half the mainloop's rate on H100).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}

// Every wait in this repo goes through here.  A pipeline bug would otherwise hang the GPU; the
// watchdog turns it into a trap (cudaErrorLaunchFailure on the host) after ~4 s of spinning.  The trap
// is inline: a function call here would make ptxas serialise every wgmma of the calling kernel.
#ifndef TC05_WATCHDOG_CYCLES
#define TC05_WATCHDOG_CYCLES 8000000000ll
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  (void)tag;   // call-site id: not reported, since printing it needs a call (above); each call site has its own trap
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0 && clock64() - t0 > TC05_WATCHDOG_CYCLES) asm volatile("trap;");
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// 2-D tiled load, completes `box bytes` on `bar` (OOB elements are zero-filled and still counted).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                            int c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(hint)
      : "memory");
}

// Same, written to the same smem offset of every CTA of the cluster named by `cta_mask`; the bytes
// complete on the barrier at the same offset in each of those CTAs.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                                      int c1, uint16_t cta_mask, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(cta_mask), "l"(hint)
      : "memory");
}

// 2-D tiled store smem -> global (bulk async group; rows/cols outside the tensor are clipped)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the bulk groups of this thread have finished READING shared memory (it may be reused)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// per-thread register budget of the calling warpgroup (all 128 threads execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ----------------------------------------------------------------------------------------------
// wgmma: descriptors
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor for a K-major operand tile stored as rows of 128 bytes
// (64 x 16-bit) with the 128-byte swizzle (what a TMA box {64, rows} with SWIZZLE_128B writes).
//   bits [ 0,14) start address >> 4      bits [16,30) leading byte offset >> 4 (unused here: 1)
//   bits [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024)
//   bits [49,52) base offset = 0 (tile base is 1024-B aligned)      bits [62,64) layout = 1 (SW128)
// A K step of 16 elements inside the 128-byte span advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Shared-memory descriptor for an MN-major operand (the MN dimension is contiguous): tile stored
// as `k` rows of 128 bytes (64 x 16-bit along MN) with the 128-byte swizzle, i.e. a TMA box
// {64 (mn), k rows}.  Canonical layout ((8,m),(8,k)) in 16-B units: 8-row (k) groups are
// `sbo_bytes` apart, successive 64-element MN blocks are `lbo_bytes` apart.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                       uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

enum : uint32_t { kFmtF16 = 0, kFmtBF16 = 1 };

// ----------------------------------------------------------------------------------------------
// wgmma: issue / commit / wait.  All 128 threads of a warpgroup execute these together.
// Accumulator fragment of m64nN (f32): thread t of the warpgroup holds, for j in [0, N/8),
//   d[4j + 0..1] = D[16 (t/32) + (t%32)/4    ][8j + 2 (t%4) + 0..1]
//   d[4j + 2..3] = D[16 (t/32) + (t%32)/4 + 8][8j + 2 (t%4) + 0..1]
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// operand lists of m64nNk16 with fp32 accumulators: N/2 registers per thread
#define TC05_R8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define TC05_R32 TC05_R8(0), TC05_R8(8), TC05_R8(16), TC05_R8(24)
#define TC05_R64 TC05_R32, TC05_R8(32), TC05_R8(40), TC05_R8(48), TC05_R8(56)
#define TC05_S32                                                                  \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "        \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define TC05_S64                                                                  \
  TC05_S32 ", "                                                                   \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define TC05_R128 TC05_R64, TC05_R8(64), TC05_R8(72), TC05_R8(80), TC05_R8(88), TC05_R8(96), TC05_R8(104), TC05_R8(112), TC05_R8(120)
#define TC05_S128                                                                               \
  TC05_S64 ", "                                                                                 \
  "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "            \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "            \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
// NAME, PTX shape + types, accumulator registers, their operand strings / constraints, operand numbers of the inputs
#define TC05_WGMMA(NAME, INSTR, NR, SLIST, RLIST, IA, IB, IP, IT)                                                     \
  template <int kTransB>                                                                                              \
  __device__ __forceinline__ void NAME(float (&d)[NR], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {        \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" IP ", 0;\n\t" INSTR " {" SLIST "}, %" IA ", %" IB           \
                 ", p, 1, 1, 0, %" IT ";\n\t}"                                                                        \
                 : RLIST                                                                                              \
                 : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransB));                                            \
  }
TC05_WGMMA(wgmma_m64n256k16_bf16, "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16", 128, TC05_S128, TC05_R128, "128", "129", "130", "131")
TC05_WGMMA(wgmma_m64n256k16_f16, "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16", 128, TC05_S128, TC05_R128, "128", "129", "130", "131")
TC05_WGMMA(wgmma_m64n128k16_bf16,"wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", 64, TC05_S64, TC05_R64, "64", "65", "66", "67")
TC05_WGMMA(wgmma_m64n128k16_f16, "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16", 64, TC05_S64, TC05_R64, "64", "65", "66", "67")
TC05_WGMMA(wgmma_m64n64k16_bf16, "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16", 32, TC05_S32, TC05_R32, "32", "33", "34", "35")
TC05_WGMMA(wgmma_m64n64k16_f16, "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16", 32, TC05_S32, TC05_R32, "32", "33", "34", "35")

// D (+)= A[smem] * B[smem], m64 x N x k16; kTransB = 1: B is MN-major
template <uint32_t FMT, int kTransB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (FMT == kFmtBF16) wgmma_m64n256k16_bf16<kTransB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n256k16_f16<kTransB>(d, adesc, bdesc, accumulate);
}
template <uint32_t FMT, int kTransB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (FMT == kFmtBF16) wgmma_m64n128k16_bf16<kTransB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n128k16_f16<kTransB>(d, adesc, bdesc, accumulate);
}
template <uint32_t FMT, int kTransB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (FMT == kFmtBF16) wgmma_m64n64k16_bf16<kTransB>(d, adesc, bdesc, accumulate);
  else wgmma_m64n64k16_f16<kTransB>(d, adesc, bdesc, accumulate);
}

// D += A[registers] * B[smem], m64n64k16, B MN-major.  A fragment (4 x 32-bit, two 16-bit values each, low half = lower
// k): thread t holds rows 16 (t/32) + (t%32)/4 (+8) and k = 2 (t%4) + 0..1 (+8), i.e. a[0] = (row, k), a[1] = (row + 8,
// k), a[2] = (row, k + 8), a[3] = (row + 8, k + 8): the accumulator fragment of an m64nN tile, columns [16 s, 16 s + 16),
// packed in pairs, is the A fragment of k step s.
#define TC05_WGMMA_RS(NAME, INSTR)                                                                                    \
  __device__ __forceinline__ void NAME(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {                     \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t" INSTR " {" TC05_S32                              \
                 "}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"                                                     \
                 : TC05_R32                                                                                           \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1u));                                  \
  }
TC05_WGMMA_RS(wgmma_m64n64k16_rs_bf16, "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16")
TC05_WGMMA_RS(wgmma_m64n64k16_rs_f16, "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16")
template <uint32_t FMT>
__device__ __forceinline__ void wgmma_n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (FMT == kFmtBF16) wgmma_m64n64k16_rs_bf16(d, a, bdesc);
  else wgmma_m64n64k16_rs_f16(d, a, bdesc);
}
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(uint32_t (&a)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(a[i])::"memory");
}


// ----------------------------------------------------------------------------------------------
// accumulator tiles in shared memory: fp32, row-major, `pitch` words per row (pitch % 32 == 4: the
// row-per-thread reads below are free of bank conflicts).  The wgmma fragment of rows [r0, r0 + 64) is
// written by its warpgroup; afterwards any thread reads whole 32-column chunks of one row.
// ----------------------------------------------------------------------------------------------
template <int R>
__device__ __forceinline__ void acc_store_frag(float* tile, int pitch, int r0, int c0, const float (&d)[R]) {
  const int t = threadIdx.x & 127;
  const int r = r0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c = c0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(tile + r * pitch + c + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(tile + (r + 8) * pitch + c + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// 32 consecutive fp32 accumulator words at shared-memory WORD address `waddr` (byte address / 4)
__device__ __forceinline__ void acc_ld_x32(uint32_t waddr, uint32_t* v) {
#pragma unroll
  for (int i = 0; i < 32; i += 4)
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[i]), "=r"(v[i + 1]), "=r"(v[i + 2]), "=r"(v[i + 3])
                 : "r"((waddr + i) * 4u)
                 : "memory");
}

// ----------------------------------------------------------------------------------------------
// ring-buffer bookkeeping
// ----------------------------------------------------------------------------------------------
template <int kStages>
struct Ring {
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
};

}  // namespace tc05

// ----------------------------------------------------------------------------------------------
// host: tensor-map encode through the driver entry point (no link-time libcuda dependency)
// ----------------------------------------------------------------------------------------------
namespace tc05_host {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D row-major 16-bit matrix [rows, cols] with row pitch `ld_elems`; box = {64 cols, box_rows},
// 128-byte swizzle.  Returns false on failure.
inline bool make_tmap_2d_16b(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                             uint32_t box_rows, uint32_t box_cols = 64) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

}  // namespace tc05_host
