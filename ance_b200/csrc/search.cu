// search.cu — flat inner-product top-k search on sm_90a.
//
// Replaces faiss.IndexFlatIP(dim).add / .search as called by the reference at
//   drivers/run_ann_data_gen.py:269-276,303 and drivers/run_ann_data_gen_dpr.py:238-252.
//
// Pipeline of one ance_index_search (all on the caller's stream):
//   1. quantize_rows_kernel : Q fp32 -> 16-bit operands (+ ||q^||, ||q - q^|| per query)
//   2. tc05_gemm_kernel<EpTopK> : coarse scores Q^ * P^^T on the tensor cores (wgmma, accumulator tile
//      in shared memory); the epilogue never stores scores — every thread owns one query row, filters
//      the 128 x BN tile against that query's running threshold and appends survivors to a
//      per-query reservoir that a warp-cooperative radix select compacts to the best k'.
//   3. rescore_kernel : exact scores (fp32 inputs, fp64 accumulate, one rounding to fp32) of the
//      <= n_splits * k' candidates, sort by (score desc, row asc), emit top-k, and CERTIFY: every
//      row that was not a candidate has coarse score <= thr, hence exact score <= thr + eps(q);
//      if thr + eps(q) < k-th exact score the result is provably the exact top-k.
//   4. tier 2, for the queries step 3 could not certify: the SAME coarse kernel once more over those queries only,
//      started from a per-query threshold t(q) = s_k - eps(q) (s_k = k-th exact score found so far, a lower bound of
//      the true one).  Every row that can still belong to the top-k has coarse score > t(q), so unless more than
//      ~2000 rows per split sit within eps of the boundary nothing is dropped and the result is certified BY
//      CONSTRUCTION: a failed certificate costs one more coarse pass over the failed queries, not a brute force.
//   5. exact_* kernels : what is left (thousands of near-ties at the boundary: duplicated rows, adversarial data) is
//      recomputed by brute force in exact arithmetic.  Also the validation path (ance_index_search_exact).
#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.h"
#include "gemm_core.cuh"

namespace {

using namespace tc05;

// ------------------------------------------------------------------------------------------------
// order-preserving float <-> uint32 (larger float -> larger key)
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f2ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
#endif
  return u ^ (static_cast<uint32_t>(static_cast<int32_t>(u) >> 31) | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
// 64-bit sort key: score descending, then row ascending  (larger key = better)
__device__ __forceinline__ uint64_t make_key(float score, uint32_t row) {
  return (static_cast<uint64_t>(f2ord(score)) << 32) | static_cast<uint64_t>(0xFFFFFFFFu - row);
}
__device__ __forceinline__ float key_score(uint64_t k) { return ord2f(static_cast<uint32_t>(k >> 32)); }
__device__ __forceinline__ uint32_t key_row(uint64_t k) { return 0xFFFFFFFFu - static_cast<uint32_t>(k); }

template <class T>
__device__ __forceinline__ T* shfl_ptr(T* p, int src) {
  uint64_t v = reinterpret_cast<uint64_t>(p);
  uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return reinterpret_cast<T*>((static_cast<uint64_t>(hi) << 32) | lo);
}

// ------------------------------------------------------------------------------------------------
// 1. fp32 -> 16-bit operand rows, with the norms the certificate needs
// ------------------------------------------------------------------------------------------------
// mu (index rows only, may be null): the rows are CENTRED before rounding, x' = x - mu.  <q, x> = <q, x - mu> + <q, mu> and
// the second term is the same for every row, so the ranking is unchanged while every norm in the certificate's error bound
// becomes that of the centred row — embeddings that share a large common component (anisotropic BERT-style outputs, an
// untrained / collapsed encoder) would otherwise spend the 16-bit significand on the component that cannot change the order.
template <bool kBF16>
__global__ void quantize_rows_kernel(const float* __restrict__ X, uint16_t* __restrict__ X16, int64_t n, int d,
                                     const float* __restrict__ mu, float* __restrict__ norm_hat,
                                     float* __restrict__ norm_delta, unsigned int* __restrict__ max_stats,
                                     int* __restrict__ err_flag) {
  // err_flag: set to 1 when a value is non-finite after rounding (fp16 overflow, or inf / NaN in the input)
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const float* x = X + row * d;
  uint16_t* o = X16 + row * d;
  float sh = 0.f, sd = 0.f, sx = 0.f;
  bool bad = false;
  for (int i = lane * 4; i < d; i += 128) {  // d % 4 == 0 (checked on the host)
    float4 v = __ldg(reinterpret_cast<const float4*>(x + i));
    if (mu) {
      const float4 m = __ldg(reinterpret_cast<const float4*>(mu + i));
      v.x -= m.x; v.y -= m.y; v.z -= m.z; v.w -= m.w;
    }
    float a[4] = {v.x, v.y, v.z, v.w};
    uint16_t q[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float back;
      if (kBF16) {
        __nv_bfloat16 h = __float2bfloat16_rn(a[t]);
        q[t] = __bfloat16_as_ushort(h);
        back = __bfloat162float(h);
      } else {
        __half h = __float2half_rn(a[t]);
        q[t] = __half_as_ushort(h);
        back = __half2float(h);
      }
      if (!(fabsf(back) <= 3.0e38f)) bad = true;  // inf / nan after rounding
      sh = fmaf(back, back, sh);
      const float e = a[t] - back;
      sd = fmaf(e, e, sd);
      sx = fmaf(a[t], a[t], sx);
    }
    uint2 pk;
    pk.x = static_cast<uint32_t>(q[0]) | (static_cast<uint32_t>(q[1]) << 16);
    pk.y = static_cast<uint32_t>(q[2]) | (static_cast<uint32_t>(q[3]) << 16);
    *reinterpret_cast<uint2*>(o + i) = pk;
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    sh += __shfl_xor_sync(0xffffffffu, sh, s);
    sd += __shfl_xor_sync(0xffffffffu, sd, s);
    sx += __shfl_xor_sync(0xffffffffu, sx, s);
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0 && err_flag) atomicExch(err_flag, 1);
  if (lane == 0) {
    // round the bounds up a little: they are upper bounds in the certificate
    // (the fp32 subtraction x - mu is itself rounded: at most 2^-24 |x - mu| per element, charged to the delta norm)
    const float nh = sqrtf(sh) * 1.00001f, nd = (sqrtf(sd) + (mu ? 1.2e-7f * sqrtf(sx) : 0.f)) * 1.00001f;
    if (norm_hat) norm_hat[row] = nh;
    if (norm_delta) norm_delta[row] = nd;
    if (max_stats) {  // non-negative floats order like their bit patterns
      atomicMax(&max_stats[0], __float_as_uint(nh));
      atomicMax(&max_stats[1], __float_as_uint(nd));
    }
  }
}

// column sums of a slab of rows (fp64), one atomicAdd per (block, column); then mu = sums / n
__global__ void __launch_bounds__(256) column_sum_kernel(const float* __restrict__ X, int64_t n, int d, int slab,
                                                         double* __restrict__ sums) {
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * slab, r1 = min(n, r0 + slab);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    double acc = 0.0;
    for (int64_t r = r0; r < r1; ++r) acc += static_cast<double>(__ldg(X + r * d + c));
    atomicAdd(sums + c, acc);
  }
}
__global__ void finalize_mean_kernel(const double* __restrict__ sums, int64_t n, int d, float* __restrict__ mu) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < d) mu[c] = static_cast<float>(sums[c] / static_cast<double>(n));
}

// ------------------------------------------------------------------------------------------------
// 2. coarse pass epilogue: per-query running top-k' over the swept corpus tiles
// ------------------------------------------------------------------------------------------------
// kStream = false: compaction holds the reservoir in registers (CAP / 32 keys and ids per lane; CAP <= 2048).
// kStream = true (EpTopKWide, reservoirs of 8192 for k > 512): compaction streams over the reservoir in memory with an
// 8-bit-digit radix select whose histograms live in the epilogue's shared memory (one 256-bin histogram per epilogue
// warp), so no register array grows with CAP.
template <int BN, int CAP, bool kStream = false>
struct EpTopK {
  static constexpr uint64_t kHintA = tc05::kEvictLast;   // query tile: re-read for every corpus tile
  static constexpr uint64_t kHintB = tc05::kEvictNormal;  // corpus rows: every concurrently sweeping CTA pair re-reads
                                                          // the same tile from L2 (EVICT_FIRST would make each pair
                                                          // stream the whole operand from HBM by itself)
  static constexpr int kEpiWarps = 4;   // the coarse pass launches 4 epilogue warps (launch_coarse)
  static constexpr int kSmemBytes = kStream ? kEpiWarps * 256 * 4 : 0;
  struct Params {
    float* scratch_sc;  // [gridDim.x * 128 * CAP] reservoir scores
    int* scratch_id;    // [gridDim.x * 128 * CAP] reservoir rows
    int* cand_id;       // [nq * n_splits * out_cap]
    int* cand_cnt;      // [nq * n_splits]
    float* cand_thr;    // [nq * n_splits]  final running threshold: every row NOT in the candidate list has coarse score <= it
    const float* thr_init;  // [nq] starting threshold per query (tier 2), or null: -inf
    int kprime;         // a reservoir that fills up is compacted to its best kprime entries
    int out_cap;        // entries kept per (query, split) at the end: kprime (tier 1) or the reservoir size (tier 2: nothing
                        // that passed the threshold is dropped unless the reservoir itself overflowed)
    int nq, n_rows;
  };

  float thr;
  int cnt;
  float* sc;
  int* id;

  __device__ __forceinline__ void begin_work(const Params& p, const gemm::WorkShape&, const gemm::EpiCtx& cx) {
    const int r = cx.quad * 32 + cx.lane;
    const size_t base = (static_cast<size_t>(blockIdx.x) * gemm::BM + r) * CAP;
    sc = p.scratch_sc + base;
    id = p.scratch_id + base;
    thr = (cx.row0 + r < p.nq) ? (p.thr_init ? __ldg(p.thr_init + cx.row0 + r) : -INFINITY) : INFINITY;
    cnt = 0;
  }

  // Warp-cooperative exact selection of the best kprime entries of lane `src`'s reservoir
  // (radix select on the order-preserving key, stable compaction: among equal scores the earlier
  // = lower row wins).  Afterwards src.cnt = kprime and src.thr = kprime-th best coarse score.
  __device__ __forceinline__ void compact(int kprime, int src, const gemm::EpiCtx& cx) {
    if constexpr (kStream) compact_stream(kprime, src, cx);
    else compact_regs(kprime, src, cx.lane);
  }

  __device__ __forceinline__ void compact_regs(int kprime, int src, int lane) {
    constexpr int kSlots = CAP / 32;
    const int n = __shfl_sync(0xffffffffu, cnt, src);
    float* s_sc = shfl_ptr(sc, src);
    int* s_id = shfl_ptr(id, src);
    uint32_t keys[kSlots];
    int ids[kSlots];
#pragma unroll
    for (int j = 0; j < kSlots; ++j) {
      const int i = j * 32 + lane;
      const bool v = i < n;
      keys[j] = v ? f2ord(s_sc[i]) : 0u;
      ids[j] = v ? s_id[i] : -1;
    }
    uint32_t prefix = 0;
    int remaining = kprime;
#pragma unroll 1
    for (int b = 31; b >= 0; --b) {
      const uint32_t cand = prefix | (1u << b);
      const uint32_t mask = ~((1u << b) - 1u);
      int c = 0;
#pragma unroll
      for (int j = 0; j < kSlots; ++j) c += ((keys[j] & mask) == cand) ? 1 : 0;
      c = __reduce_add_sync(0xffffffffu, c);
      if (c >= remaining) prefix = cand;
      else remaining -= c;
    }
    const uint32_t T = prefix;
    const unsigned lt = (1u << lane) - 1u;
    int base = 0, eq_seen = 0;
#pragma unroll
    for (int j = 0; j < kSlots; ++j) {
      const bool gt = keys[j] > T, eq = keys[j] == T;
      const unsigned eqm = __ballot_sync(0xffffffffu, eq);
      const bool keep = gt || (eq && (eq_seen + __popc(eqm & lt)) < remaining);
      const unsigned km = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int pos = base + __popc(km & lt);
        s_sc[pos] = ord2f(keys[j]);
        s_id[pos] = ids[j];
      }
      base += __popc(km);
      eq_seen += __popc(eqm);
    }
    __syncwarp();
    if (lane == src) {
      cnt = kprime;
      thr = ord2f(T);
    }
  }

  // Same contract as compact_regs, for reservoirs too large for registers.  Four passes over lane `src`'s reservoir
  // build 8-bit digit histograms (most significant digit first, only keys that match the digits chosen so far) and pick
  // the digit that holds the kprime-th best key; a fifth pass compacts in place, stably.  In place is safe: every lane
  // reads its entry of a 32-entry chunk before any lane writes (the ballots order them), and the write position never
  // exceeds the read position.
  __device__ __forceinline__ void compact_stream(int kprime, int src, const gemm::EpiCtx& cx) {
    const int lane = cx.lane;
    const int n = __shfl_sync(0xffffffffu, cnt, src);
    float* s_sc = shfl_ptr(sc, src);
    int* s_id = shfl_ptr(id, src);
    uint32_t* hist = reinterpret_cast<uint32_t*>(cx.ep_smem) + cx.epi_warp * 256;
    uint32_t prefix = 0;
    int remaining = kprime;   // keys still to select among those that match `prefix`
#pragma unroll 1
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = lane; b < 256; b += 32) hist[b] = 0u;
      __syncwarp();
      const uint32_t hmask = (shift == 24) ? 0u : ~((1u << (shift + 8)) - 1u);   // the digits already chosen
      for (int i = lane; i < n; i += 32) {
        const uint32_t key = f2ord(s_sc[i]);
        if ((key & hmask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
      __syncwarp();
      // lane l owns digits 255 - 8l down to 248 - 8l: an exclusive scan over lanes counts the keys of larger digits
      uint32_t c[8];
      int sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[255 - (lane * 8 + j)];
        sum += static_cast<int>(c[j]);
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const int excl = incl - sum;
      const unsigned owner = __ballot_sync(0xffffffffu, excl < remaining && remaining <= incl);
      const int ol = __ffs(owner) - 1;
      int digit = -1, above = 0, acc = excl;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (digit < 0 && acc + static_cast<int>(c[j]) >= remaining) {
          digit = 255 - (lane * 8 + j);
          above = acc;
        }
        acc += static_cast<int>(c[j]);
      }
      digit = __shfl_sync(0xffffffffu, digit, ol);
      above = __shfl_sync(0xffffffffu, above, ol);
      prefix |= static_cast<uint32_t>(digit) << shift;
      remaining -= above;
      __syncwarp();
    }
    const uint32_t T = prefix;   // the kprime-th best key; keep every larger key and the first `remaining` equal ones
    const unsigned lt = (1u << lane) - 1u;
    int base = 0, eq_seen = 0;
#pragma unroll 1
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const bool v = i < n;
      const float s = v ? s_sc[i] : 0.f;
      const int r = v ? s_id[i] : 0;
      const uint32_t key = f2ord(s);
      const bool gt = v && key > T, eq = v && key == T;
      const unsigned eqm = __ballot_sync(0xffffffffu, eq);
      const bool keep = gt || (eq && (eq_seen + __popc(eqm & lt)) < remaining);
      const unsigned km = __ballot_sync(0xffffffffu, keep);
      __syncwarp();   // every read of this chunk before any write into it
      if (keep) {
        const int pos = base + __popc(km & lt);
        s_sc[pos] = s;
        s_id[pos] = r;
      }
      base += __popc(km);
      eq_seen += __popc(eqm);
    }
    __syncwarp();
    if (lane == src) {
      cnt = kprime;
      thr = ord2f(T);
    }
  }

  __device__ __forceinline__ void tile(const Params& p, const gemm::WorkShape&, const gemm::EpiCtx& cx,
                                       uint32_t tacc, int nb) {
#pragma unroll 1
    for (int c = 0; c < BN; c += 32) {
      uint32_t v[32];
      acc_ld_x32(tacc + c, v);
      float m = __uint_as_float(v[0]);
#pragma unroll
      for (int i = 1; i < 32; ++i) m = fmaxf(m, __uint_as_float(v[i]));
      if (m > thr) {
        const int col0 = nb * BN + c;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float s = __uint_as_float(v[i]);
          if (s > thr && col0 + i < p.n_rows) {  // rows past the end are TMA zero fill
            sc[cnt] = s;
            id[cnt] = col0 + i;
            ++cnt;
          }
        }
      }
      __syncwarp();
      unsigned need = __ballot_sync(0xffffffffu, cnt > CAP - 32);
      while (need) {
        const int src = __ffs(need) - 1;
        need &= need - 1;
        compact(p.kprime, src, cx);
      }
    }
  }

  __device__ __forceinline__ void end_kernel(const Params&, const gemm::EpiCtx&) {}

  __device__ __forceinline__ void end_work(const Params& p, const gemm::WorkShape& ws, const gemm::EpiCtx& cx) {
    __syncwarp();
    unsigned need = __ballot_sync(0xffffffffu, cnt > p.out_cap);
    while (need) {
      const int src = __ffs(need) - 1;
      need &= need - 1;
      compact(p.kprime, src, cx);
    }
    for (int l = 0; l < 32; ++l) {
      const int row = cx.row0 + cx.quad * 32 + l;
      if (row >= p.nq) break;  // warp-uniform
      const int n = __shfl_sync(0xffffffffu, cnt, l);
      const float t = __shfl_sync(0xffffffffu, thr, l);
      const int* s_id = shfl_ptr(id, l);
      const size_t slot = static_cast<size_t>(row) * ws.n_splits + cx.split;
      int* out = p.cand_id + slot * p.out_cap;
      for (int i = cx.lane; i < n; i += 32) out[i] = s_id[i];
      if (cx.lane == 0) {
        p.cand_cnt[slot] = n;
        p.cand_thr[slot] = t;
      }
    }
    __syncwarp();
  }
};

// ------------------------------------------------------------------------------------------------
// shared helpers: exact dot products and block bitonic sort
// ------------------------------------------------------------------------------------------------
// Loads of fp32 index rows.  kHost: the rows are pinned host memory mapped into the device's address space (a host
// index): plain ld.global, never the non-coherent read-only path.  Otherwise __ldg, as the device index always had.
template <bool kHost>
__device__ __forceinline__ float4 ld_rows4(const float* p) {
  if constexpr (kHost) {
    float4 v;
    asm("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
  } else {
    return __ldg(reinterpret_cast<const float4*>(p));
  }
}
template <bool kHost>
__device__ __forceinline__ float ld_rows1(const float* p) {
  if constexpr (kHost) {
    float v;
    asm("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
  } else {
    return __ldg(p);
  }
}

// exact <q, p>: fp32 inputs, products and sum in fp64 (each product is exact in fp64), result
// rounded once to fp32.  Lane-strided float4 loads; deterministic shuffle tree.
template <bool kHost = false>
__device__ __forceinline__ double warp_dot_f64(const float* __restrict__ q_smem, const float* __restrict__ p, int d,
                                               int lane) {
  double acc = 0.0;
  if ((d & 127) == 0) {
    for (int i = lane * 4; i < d; i += 128) {
      const float4 a = *reinterpret_cast<const float4*>(q_smem + i);
      const float4 b = ld_rows4<kHost>(p + i);
      acc = fma(static_cast<double>(a.x), static_cast<double>(b.x), acc);
      acc = fma(static_cast<double>(a.y), static_cast<double>(b.y), acc);
      acc = fma(static_cast<double>(a.z), static_cast<double>(b.z), acc);
      acc = fma(static_cast<double>(a.w), static_cast<double>(b.w), acc);
    }
  } else {
    for (int i = lane; i < d; i += 32) acc = fma(static_cast<double>(q_smem[i]), static_cast<double>(ld_rows1<kHost>(p + i)), acc);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
  return acc;
}

// descending bitonic sort of n (power of two) 64-bit keys in shared memory by the whole block
__device__ __forceinline__ void block_bitonic_desc(uint64_t* keys, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const uint64_t a = keys[lo], b = keys[hi];
        if ((a < b) == desc) {
          keys[lo] = b;
          keys[hi] = a;
        }
      }
    }
  }
  __syncthreads();
}

__host__ __device__ inline int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// ------------------------------------------------------------------------------------------------
// 3. exact rescoring of the candidates + certificate
// ------------------------------------------------------------------------------------------------
struct RescoreParams {
  const float* Q;
  const float* P;
  int d;
  const int* cand_id;
  const int* cand_cnt;
  const float* cand_thr;
  int n_splits, cand_stride, k;   // cand_stride = EpTopK out_cap
  const float* qn_hat;
  const float* qn_delta;
  const unsigned int* pstats;  // [0] max ||p^||, [1] max ||p - p^|| (float bits) of the CENTRED rows
  const float* mu;             // the centre subtracted from every index row before rounding (null: none)
  float accum_rel;             // bound on the tensor core's accumulation error / (||q^|| ||p^||), see coarse_rescore_pass
  float* D;
  int64_t* I;
  int64_t row_offset;
  const int* qlist;    // block b handles candidate slot b of query qlist[b] (null: query b)
  int* flagged_list;   // uncertified queries of this pass
  float* flagged_thr;  // starting threshold of the next tier for flagged_list[i] (null: not needed)
  int flag_slot;       // counters[flag_slot] counts them
  int* counters;       // [0] tier-1 flagged [1] n_candidates [2] max eps bits [3] tier-2 flagged
  unsigned int* max_eps;
  int sort_n;          // pow2 >= total candidates of a query
  // host index only (rescore_kernel<true>): the pre-filter's inputs
  const uint16_t* P16;      // [n, d] 16-bit operand rows (centred, rounded)
  const float* ndelta;      // [n] ||p_j - mu - p^_j|| per row, rounded up
  int bf16;                 // operand format of P16
};

constexpr int kCntFetched = 4;   // counters[4]: rows rescoring read from host memory (host index)

// exact <q, p_c> of kNB candidate rows at once: all the row's 16-byte loads (d / 128 per lane and row) are issued
// before the first fp64 FMA, so a warp keeps kNB * d / 128 gathers in flight instead of one (the rows are random
// 3 KB reads: latency, not bandwidth, bounded the one-row-at-a-time form at 0.14 of HBM).  kJ = d / 128 (768: kJ = 6).
template <int kNB, int kJ, bool kHost = false>
__device__ __forceinline__ void warp_dots_f64(const float* __restrict__ q_smem, const float* const (&rows)[kNB], int d,
                                              int lane, double (&out)[kNB]) {
  float4 b[kNB][kJ];
#pragma unroll
  for (int j = 0; j < kJ; ++j) {
    {
#pragma unroll
      for (int c = 0; c < kNB; ++c) b[c][j] = ld_rows4<kHost>(rows[c] + j * 128 + lane * 4);
    }
  }
#pragma unroll
  for (int c = 0; c < kNB; ++c) out[c] = 0.0;
#pragma unroll
  for (int j = 0; j < kJ; ++j) {
    {
      const float4 a = *reinterpret_cast<const float4*>(q_smem + j * 128 + lane * 4);
#pragma unroll
      for (int c = 0; c < kNB; ++c) {   // same association as warp_dot_f64: the result is bit-identical
        out[c] = fma(static_cast<double>(a.x), static_cast<double>(b[c][j].x), out[c]);
        out[c] = fma(static_cast<double>(a.y), static_cast<double>(b[c][j].y), out[c]);
        out[c] = fma(static_cast<double>(a.z), static_cast<double>(b[c][j].z), out[c]);
        out[c] = fma(static_cast<double>(a.w), static_cast<double>(b[c][j].w), out[c]);
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int c = 0; c < kNB; ++c) out[c] += __shfl_xor_sync(0xffffffffu, out[c], s);
  }
}

// order-preserving double -> uint64 (larger double -> larger key; every non-NaN value maps above 0)
__device__ __forceinline__ uint64_t d2ord(double x) {
  const uint64_t u = static_cast<uint64_t>(__double_as_longlong(x));
  return u ^ (static_cast<uint64_t>(static_cast<int64_t>(u) >> 63) | 0x8000000000000000ull);
}
__device__ __forceinline__ double ord2d(uint64_t k) {
  return __longlong_as_double(static_cast<long long>((k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k));
}

// Candidate scores of a HOST index (rows in pinned host memory, every fp32 row read crosses PCIe): a pre-filter on data
// in HBM, then exact scores of the survivors only.  Writes keys[pos] of every candidate position (0 for a pruned one).
//   Phase A: s~_j = <q, p^_j> in fp64 from the 16-bit operand row (the products are exact in fp64), and
//            lo_j / hi_j = <q, mu> + s~_j -/+ (||q|| ||delta_j|| + g), so lo_j <= <q, p_j> <= hi_j; g bounds the fp64
//            summation error of one dot product over d terms, (d + 16) 2^-53 ||q|| ||p||, for every row (DESIGN.md §4.2).
//            L = k-th largest lo.
//   Phase B: prune j iff fl32_up(hi_j + g) < fl32_down(L - g), and compute the exact score of every other candidate
//            (the same warp_dots_f64 association as the device index: bit-identical scores).
// At least k candidates score >= fl32_down(L - g) and a pruned row scores <= fl32_up(hi_j + g), strictly less: the top k
// of the survivors are the top k of all candidates, ties included, and the certificate sees the same k-th score.
// extra: 16 * sort_n bytes of shared memory (hi [sort_n] fp64, rows [sort_n], survivors [sort_n]).
__device__ __forceinline__ void host_rows_scores(const RescoreParams& p, uint64_t* keys, const float* qs, const int* offs,
                                              const double* s_qmu, uint8_t* extra, int ql) {
  double* hi = reinterpret_cast<double*>(extra);
  int* rows = reinterpret_cast<int*>(hi + p.sort_n);
  int* surv = rows + p.sort_n;
  __shared__ double s_red[2][8];
  __shared__ double s_g;
  __shared__ double s_qn;
  __shared__ double s_base;
  __shared__ float s_T;
  __shared__ int s_nsurv;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int d = p.d, m = offs[p.n_splits];
  double qq = 0.0, mm = 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    qq = fma(static_cast<double>(qs[i]), static_cast<double>(qs[i]), qq);
    if (p.mu) mm = fma(static_cast<double>(__ldg(p.mu + i)), static_cast<double>(__ldg(p.mu + i)), mm);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    qq += __shfl_xor_sync(0xffffffffu, qq, s);
    mm += __shfl_xor_sync(0xffffffffu, mm, s);
  }
  if (lane == 0) {
    s_red[0][warp] = qq;
    s_red[1][warp] = mm;
  }
  for (int s = 0; s < p.n_splits; ++s) {
    const int* ids = p.cand_id + (static_cast<size_t>(ql) * p.n_splits + s) * p.cand_stride;
    for (int c = threadIdx.x; c < offs[s + 1] - offs[s]; c += blockDim.x) rows[offs[s] + c] = ids[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sq = 0.0, sm = 0.0, qmu = 0.0;
    for (int w = 0; w < nwarps; ++w) {
      sq += s_red[0][w];
      sm += s_red[1][w];
      qmu += s_qmu[w];
    }
    // every fp64 sum of d products above carries a relative error below (d + 16) 2^-53: inflate by twice that
    const double infl = 1.0 + static_cast<double>(d + 16) * 0x1p-52;
    const double qn = __dsqrt_ru(__dmul_ru(sq, infl));
    const double mun = __dsqrt_ru(__dmul_ru(sm, infl));
    const double maxp = static_cast<double>(__uint_as_float(p.pstats[0])), maxdp = static_cast<double>(__uint_as_float(p.pstats[1]));
    // g >= (d + 16) 2^-53 ||q|| ||x|| with ||x|| <= ||mu|| + max ||p^|| + max ||delta||: covers the summation error of
    // s~_j + <q, mu> (one g) and of the exact fp64 score (the other g)
    s_g = __dmul_ru(__dmul_ru(static_cast<double>(d + 16) * 0x1p-53, qn), __dadd_ru(__dadd_ru(mun, maxp), maxdp));
    s_qn = qn;
    s_base = qmu;
  }
  __syncthreads();
  const double g = s_g, qn = s_qn, qmu = s_base;
  // ||delta_j|| is an fp32 sum of d squares (+ sqrt): charge its relative rounding error once more
  const double nd_infl = 1.0 + static_cast<double>(d + 64) * 0x1p-23;
  // --- phase A: bounds from the 16-bit rows in HBM
  for (int c = warp; c < m; c += nwarps) {
    const int row = rows[c];
    const uint16_t* r16 = p.P16 + static_cast<size_t>(row) * d;
    double acc = 0.0;
    for (int i = lane * 8; i < d; i += 256) {   // d % 8 == 0 (checked at creation)
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(r16 + i));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      // the lane's 8 query values as two 16-byte shared loads (a warp reads 1 KB contiguously: no bank conflicts)
      const float4 qa = *reinterpret_cast<const float4*>(qs + i), qb = *reinterpret_cast<const float4*>(qs + i + 4);
      const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const uint16_t h = static_cast<uint16_t>(w[t >> 1] >> ((t & 1) * 16));
        const float x = p.bf16 ? __uint_as_float(static_cast<uint32_t>(h) << 16) : __half2float(__ushort_as_half(h));
        acc = fma(static_cast<double>(qv[t]), static_cast<double>(x), acc);
      }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if (lane == 0) {
      const double r = __dadd_ru(__dmul_ru(qn, __dmul_ru(static_cast<double>(__ldg(p.ndelta + row)), nd_infl)), g);
      keys[c] = d2ord(__dadd_rd(__dadd_rd(qmu, acc), -r));
      hi[c] = __dadd_ru(__dadd_ru(qmu, acc), r);
    }
  }
  // L = k-th largest lo (keys past m stay 0: below every lo)
  if (m > p.k) {
    block_bitonic_desc(keys, p.sort_n);
    if (threadIdx.x == 0) s_T = __double2float_rd(__dadd_rd(ord2d(keys[p.k - 1]), -g));
  } else if (threadIdx.x == 0) {
    s_T = -INFINITY;   // at most k candidates: nothing may be pruned
  }
  if (threadIdx.x == 0) s_nsurv = 0;
  __syncthreads();
  const float T = s_T;
  for (int c = threadIdx.x; c < m; c += blockDim.x)
    if (T == -INFINITY || __double2float_ru(__dadd_ru(hi[c], g)) >= T) surv[atomicAdd(&s_nsurv, 1)] = c;
  for (int i = threadIdx.x; i < p.sort_n; i += blockDim.x) keys[i] = 0ull;
  __syncthreads();
  // --- phase B: exact scores of the survivors, fp32 rows read through the mapped host pointer
  const int ns = s_nsurv;
  constexpr int kNB = 4;
  if (d == 768) {
    for (int c0 = warp * kNB; c0 < ns; c0 += nwarps * kNB) {
      int pos[kNB];
      const float* rp[kNB];
#pragma unroll
      for (int c = 0; c < kNB; ++c) {
        pos[c] = surv[min(c0 + c, ns - 1)];
        rp[c] = p.P + static_cast<size_t>(rows[pos[c]]) * d;
      }
      double dot[kNB];
      warp_dots_f64<kNB, 6, true>(qs, rp, d, lane, dot);
      if (lane == 0) {
#pragma unroll
        for (int c = 0; c < kNB; ++c)
          if (c0 + c < ns) keys[pos[c]] = make_key(static_cast<float>(dot[c]), static_cast<uint32_t>(rows[pos[c]]));
      }
    }
  } else {
    for (int c = warp; c < ns; c += nwarps) {
      const int pos = surv[c];
      const double dot = warp_dot_f64<true>(qs, p.P + static_cast<size_t>(rows[pos]) * d, d, lane);
      if (lane == 0) keys[pos] = make_key(static_cast<float>(dot), static_cast<uint32_t>(rows[pos]));
    }
  }
  if (threadIdx.x == 0) atomicAdd(&p.counters[kCntFetched], ns);
}

template <bool kHost>
__global__ void __launch_bounds__(256) rescore_kernel(const RescoreParams p) {
  extern __shared__ __align__(16) uint8_t rs_smem[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(rs_smem);
  float* qs = reinterpret_cast<float*>(keys + p.sort_n);
  int* offs = reinterpret_cast<int*>(qs + p.d);  // [n_splits + 1]
  const int ql = blockIdx.x;                       // slot in the candidate arrays
  const int q = p.qlist ? p.qlist[ql] : ql;        // query number (rows of Q, D, I)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

  for (int i = threadIdx.x; i < p.d; i += blockDim.x) qs[i] = p.Q[static_cast<size_t>(q) * p.d + i];
  if (threadIdx.x == 0) {
    int o = 0;
    for (int s = 0; s < p.n_splits; ++s) {
      offs[s] = o;
      o += p.cand_cnt[static_cast<size_t>(ql) * p.n_splits + s];
    }
    offs[p.n_splits] = o;
  }
  __syncthreads();
  const int m = offs[p.n_splits];
  for (int i = threadIdx.x; i < p.sort_n; i += blockDim.x) keys[i] = 0ull;
  // <q, mu> in fp64: what separates the coarse (centred) scores from the exact ones, identically for every row
  __shared__ double s_qmu[8];
  {
    double part = 0.0;
    if (p.mu)
      for (int i = threadIdx.x; i < p.d; i += blockDim.x) part = fma(static_cast<double>(qs[i]), static_cast<double>(__ldg(p.mu + i)), part);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) part += __shfl_xor_sync(0xffffffffu, part, s);
    if (lane == 0) s_qmu[warp] = part;
  }
  __syncthreads();
  constexpr int kNB = 4;
  const bool wide = p.d == 768;   // the path's dimension (models.py:145-146); other dims take the one-row loop
  if constexpr (kHost) {
    const size_t extra = (static_cast<size_t>(p.sort_n) * 8 + static_cast<size_t>(p.d) * 4 + (p.n_splits + 1) * 4 + 15) & ~size_t(15);
    host_rows_scores(p, keys, qs, offs, s_qmu, rs_smem + extra, ql);
  } else
  for (int s = 0; s < p.n_splits; ++s) {
    const int n = offs[s + 1] - offs[s];
    const int* ids = p.cand_id + (static_cast<size_t>(ql) * p.n_splits + s) * p.cand_stride;
    if (wide) {
      for (int c0 = warp * kNB; c0 < n; c0 += nwarps * kNB) {
        int row[kNB];
        const float* rp[kNB];
#pragma unroll
        for (int c = 0; c < kNB; ++c) {
          row[c] = ids[min(c0 + c, n - 1)];
          rp[c] = p.P + static_cast<size_t>(row[c]) * p.d;
        }
        double dot[kNB];
        warp_dots_f64<kNB, 6>(qs, rp, p.d, lane, dot);
        if (lane == 0) {
#pragma unroll
          for (int c = 0; c < kNB; ++c)
            if (c0 + c < n) keys[offs[s] + c0 + c] = make_key(static_cast<float>(dot[c]), static_cast<uint32_t>(row[c]));
        }
      }
    } else {
      for (int c = warp; c < n; c += nwarps) {
        const int row = ids[c];
        const double dot = warp_dot_f64(qs, p.P + static_cast<size_t>(row) * p.d, p.d, lane);
        if (lane == 0) keys[offs[s] + c] = make_key(static_cast<float>(dot), static_cast<uint32_t>(row));
      }
    }
  }
  block_bitonic_desc(keys, p.sort_n);
  for (int i = threadIdx.x; i < p.k; i += blockDim.x) {
    const bool ok = i < m;
    p.D[static_cast<size_t>(q) * p.k + i] = ok ? key_score(keys[i]) : -FLT_MAX;
    p.I[static_cast<size_t>(q) * p.k + i] = ok ? p.row_offset + static_cast<int64_t>(key_row(keys[i])) : -1;
  }
  if (threadIdx.x == 0) {
    float thr = -INFINITY;
    for (int s = 0; s < p.n_splits; ++s) thr = fmaxf(thr, p.cand_thr[static_cast<size_t>(ql) * p.n_splits + s]);
    const float maxp = __uint_as_float(p.pstats[0]), maxdp = __uint_as_float(p.pstats[1]);
    const float qn = p.qn_hat[q], qd = p.qn_delta[q];
    // |coarse_j - <q, p_j>| <= eps for EVERY row j (Cauchy-Schwarz on the operand rounding + the accumulation bound);
    // the factor covers the fp32 roundings of this expression itself (norms are already rounded up)
    const float eps = (qd * maxp + qn * maxdp + qd * maxdp + p.accum_rel * qn * maxp) * 1.0001f;
    // A row that is not a candidate has centred coarse score <= thr, hence exact score <= thr + eps + <q, mu>.  The k-th
    // exact score is an fp64 dot product rounded to fp32: the unrounded value is >= sk_lo.  Compared in fp64.
    double qmu = 0.0;
    for (int w2 = 0; w2 < nwarps; ++w2) qmu += s_qmu[w2];
    const double qmu_up = qmu + fabs(qmu) * 1.0e-12;
    const double sk = (m >= p.k) ? static_cast<double>(key_score(keys[p.k - 1])) : -INFINITY;
    const double sk_lo = sk - fabs(sk) * 1.2e-7;
    bool certified;
    if (thr == -INFINITY) certified = true;       // every row of the index was a candidate
    else if (m < p.k) certified = false;          // cannot happen (thr finite => >= k candidates passed it)
    else certified = (static_cast<double>(thr) + static_cast<double>(eps) + qmu_up < sk_lo);
    atomicAdd(&p.counters[1], m);
    atomicMax(p.max_eps, __float_as_uint(eps));
    if (!certified) {
      const int slot = atomicAdd(&p.counters[p.flag_slot], 1);
      p.flagged_list[slot] = q;
      if (p.flagged_thr) {
        // Next tier starts from t < s_k - eps: every row whose exact score reaches s_k (the k-th exact score found so
        // far, a lower bound of the final one) has coarse score >= s_k - eps > t, i.e. passes the filter.
        const float x = __double2float_rd(sk_lo - qmu_up - static_cast<double>(eps));   // in centred coarse-score units
        p.flagged_thr[slot] = (m < p.k) ? -INFINITY : __fsub_rd(x, fmaxf(fabsf(x), eps) * 1.0e-6f);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 4. exact brute force (fallback for uncertified queries, and the validation path)
// ------------------------------------------------------------------------------------------------
constexpr int kExQB = 4;       // queries per block
constexpr int kExRound = 16;   // rows per warp between reservoir checks
// reservoir keys per query: must hold k + nwarps * kExRound (8 warps): 1024 for k <= 512, 4096 for k <= 2048
constexpr int kExBufSmall = 1024, kExBufLarge = 4096;

struct ExactParams {
  const float* Q;
  const float* P;
  int d;
  int64_t n_rows;
  const int* qlist;      // query numbers (null = q_base + i)
  int q_base;
  const int* nq_dev;     // number of queries on the device (null = use nq)
  int nq;
  int k;                 // <= 2048
  int n_chunks;
  uint64_t* chunk_keys;  // [nq_cap * n_chunks * k]  (run_exact_host: [nq_cap * (n_chunks + 1) * k])
};

// kSlab: p.P is a slab of a host index's rows staged in device memory (run_exact_host): keys carry the global row
// row_base + row, and every query has n_chunks + 1 key slots, the last one holding the best k of the earlier slabs.
// (row_base is a kernel argument rather than an ExactParams field, which exact_merge_kernel shares.)
template <int kExBuf, bool kSlab>
__global__ void __launch_bounds__(256) exact_chunk_kernel(const ExactParams p, int64_t row_base) {
  extern __shared__ __align__(16) uint8_t ex_smem[];
  uint64_t* buf = reinterpret_cast<uint64_t*>(ex_smem);              // [kExQB][kExBuf]
  float* qs = reinterpret_cast<float*>(buf + kExQB * kExBuf);        // [kExQB][d]
  __shared__ int cnt[kExQB];
  __shared__ unsigned long long thr[kExQB];
  const int nq = p.nq_dev ? min(*p.nq_dev, p.nq) : p.nq;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t rows_per_chunk = (p.n_rows + p.n_chunks - 1) / p.n_chunks;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * rows_per_chunk;
  const int64_t r1 = min(p.n_rows, r0 + rows_per_chunk);

  for (int g = blockIdx.y; g * kExQB < nq; g += gridDim.y) {
    const int nqb = min(kExQB, nq - g * kExQB);
    __syncthreads();
    for (int i = threadIdx.x; i < kExQB * p.d; i += blockDim.x) {
      const int qi = i / p.d, e = i - qi * p.d;
      float v = 0.f;
      if (qi < nqb) {
        const int q = p.qlist ? p.qlist[g * kExQB + qi] : p.q_base + g * kExQB + qi;
        v = p.Q[static_cast<size_t>(q) * p.d + e];
      }
      qs[i] = v;
    }
    if (threadIdx.x < kExQB) {
      cnt[threadIdx.x] = 0;
      thr[threadIdx.x] = 0ull;
    }
    __syncthreads();
    for (int64_t base = r0; base < r1; base += static_cast<int64_t>(nwarps) * kExRound) {
      for (int t = 0; t < kExRound; ++t) {
        const int64_t row = base + static_cast<int64_t>(t) * nwarps + warp;
        if (row >= r1) break;
        const float* prow = p.P + row * p.d;
        double acc[kExQB];
#pragma unroll
        for (int qi = 0; qi < kExQB; ++qi) acc[qi] = 0.0;
        for (int i = lane; i < p.d; i += 32) {
          const double b = static_cast<double>(__ldg(prow + i));
#pragma unroll
          for (int qi = 0; qi < kExQB; ++qi) acc[qi] = fma(static_cast<double>(qs[qi * p.d + i]), b, acc[qi]);
        }
#pragma unroll
        for (int qi = 0; qi < kExQB; ++qi) {
#pragma unroll
          for (int s = 16; s > 0; s >>= 1) acc[qi] += __shfl_xor_sync(0xffffffffu, acc[qi], s);
        }
        if (lane < nqb) {
          double a = acc[0];
#pragma unroll
          for (int qi = 1; qi < kExQB; ++qi)
            if (lane == qi) a = acc[qi];
          const uint64_t key = make_key(static_cast<float>(a), static_cast<uint32_t>(kSlab ? row_base + row : row));
          if (key > thr[lane]) {
            const int slot = atomicAdd(&cnt[lane], 1);
            buf[lane * kExBuf + slot] = key;  // slot < kExBuf: at most nwarps*kExRound appends per round
          }
        }
      }
      __syncthreads();
      for (int qi = 0; qi < nqb; ++qi) {
        if (cnt[qi] > kExBuf - nwarps * kExRound) {  // block-uniform
          const int n = cnt[qi];
          for (int i = n + threadIdx.x; i < kExBuf; i += blockDim.x) buf[qi * kExBuf + i] = 0ull;
          block_bitonic_desc(buf + qi * kExBuf, kExBuf);
          if (threadIdx.x == 0) {
            cnt[qi] = p.k;
            thr[qi] = buf[qi * kExBuf + p.k - 1];
          }
          __syncthreads();
        }
      }
    }
    __syncthreads();
    for (int qi = 0; qi < nqb; ++qi) {
      const int n = cnt[qi];
      for (int i = n + threadIdx.x; i < kExBuf; i += blockDim.x) buf[qi * kExBuf + i] = 0ull;
      block_bitonic_desc(buf + qi * kExBuf, kExBuf);
      uint64_t* out = p.chunk_keys + (static_cast<size_t>(g * kExQB + qi) * (kSlab ? p.n_chunks + 1 : p.n_chunks) + blockIdx.x) * p.k;
      for (int i = threadIdx.x; i < p.k; i += blockDim.x) out[i] = (i < n) ? buf[qi * kExBuf + i] : 0ull;
    }
  }
}

constexpr int kMergeBuf = 4096;   // > k: every round merges at least kMergeBuf - k new keys into the best k

// kToAcc: write the merged best k back into the query's last key slot (run_exact_host's running result) instead of D / I
template <bool kToAcc>
__global__ void __launch_bounds__(256) exact_merge_kernel(const ExactParams p, float* D, int64_t* I, int out_k,
                                                          int64_t row_offset) {
  __shared__ uint64_t keys[kMergeBuf];
  const int nq = p.nq_dev ? min(*p.nq_dev, p.nq) : p.nq;
  for (int qi = blockIdx.x; qi < nq; qi += gridDim.x) {
    const int q = p.qlist ? p.qlist[qi] : p.q_base + qi;
    const uint64_t* src = p.chunk_keys + static_cast<size_t>(qi) * p.n_chunks * p.k;
    const int total = p.n_chunks * p.k;
    int have = 0;  // keys[0..have) = current best (sorted)
    int pos = 0;
    __syncthreads();
    while (pos < total) {
      const int take = min(kMergeBuf - have, total - pos);
      for (int i = threadIdx.x; i < take; i += blockDim.x) keys[have + i] = src[pos + i];
      for (int i = have + take + threadIdx.x; i < kMergeBuf; i += blockDim.x) keys[i] = 0ull;
      pos += take;
      block_bitonic_desc(keys, kMergeBuf);
      have = p.k;
    }
    if constexpr (kToAcc) {
      uint64_t* acc = p.chunk_keys + (static_cast<size_t>(qi) * p.n_chunks + p.n_chunks - 1) * p.k;
      for (int i = threadIdx.x; i < p.k; i += blockDim.x) acc[i] = keys[i];
    } else {
    for (int i = threadIdx.x; i < out_k; i += blockDim.x) {
      const uint64_t key = (i < p.k) ? keys[i] : 0ull;
      const bool ok = key != 0ull;
      D[static_cast<size_t>(q) * out_k + i] = ok ? key_score(key) : -FLT_MAX;
      I[static_cast<size_t>(q) * out_k + i] = ok ? row_offset + static_cast<int64_t>(key_row(key)) : -1;
    }
    }
    __syncthreads();
  }
}

// 16-bit operand rows of the listed queries -> compact matrix (second, wider coarse pass)
__global__ void gather_rows16_kernel(const uint16_t* __restrict__ src, const int* __restrict__ qlist, int n, int d,
                                     uint16_t* __restrict__ dst) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(qlist[r]) * d);
  uint4* o = reinterpret_cast<uint4*>(dst + static_cast<size_t>(r) * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) o[i] = s[i];
}

}  // namespace

// ================================================================================================
// index handle
// ================================================================================================
struct ance_index {
  int dim = 0;
  int64_t cap = 0, n = 0;
  int fmt = ANCE_FMT_FP16;
  int device = 0;
  float* P32 = nullptr;      // [cap, dim]  (host index: the device address of the pinned host rows)
  bool owns_p32 = true;      // false: caller-owned storage (ance_index_create_over), or a host index
  // host index (ance_index_create_host): the fp32 rows live in pinned host memory
  bool host_rows = false;
  float* P32_host = nullptr;       // [cap, dim] host address of the rows
  bool owns_host = false;          // allocated by the library (cudaHostAlloc), freed by ance_index_destroy
  float* ndelta = nullptr;         // [cap] ||p_j - mu - p^_j|| per row (device; the rescoring pre-filter's bound)
  int64_t last_fetched = 0;        // rows the last search's rescoring read from host memory
  uint16_t* P16 = nullptr;   // [cap, dim]
  unsigned int* pstats = nullptr;  // [2]
  float* mu = nullptr;             // [dim] centre of the rows (see quantize_rows_kernel)
  double* colsum = nullptr;        // [dim]
  bool dirty = false;              // rows were added / the format changed since the 16-bit operands were (re)built
  bool centred = false;
  int center = 1;                  // tunable "center": subtract the column mean before rounding
  // tunables
  int kprime = 0, n_splits = 0, cta_group = 2, max_ctas = 0, exact_fallback = 1, tier2 = 1, pace_window = 16;
  // workspace (grown lazily)
  uint16_t* Q16 = nullptr; float* qn_hat = nullptr; float* qn_delta = nullptr; int64_t q_cap = 0;
  float* scratch_sc = nullptr; int* scratch_id = nullptr; size_t scratch_elems = 0;
  int* cand_id = nullptr; int* cand_cnt = nullptr; float* cand_thr = nullptr; size_t cand_slots = 0, cand_ids = 0;
  int* flagged = nullptr; float* flagged_thr = nullptr; int64_t flagged_cap = 0;
  int* flagged2 = nullptr; size_t flagged2_cap = 0;
  uint16_t* Q16b = nullptr; size_t q16b_elems = 0;
  int* pace = nullptr;              // [kMaxPace] progress counters of the sweeping CTA pairs (soft barrier)
  // [0] tier-1 flagged  [1] candidates rescored  [2] max eps bits  [3] tier-2 flagged  [4] rows fetched from host memory
  // [5] spare
  // [6] a QUERY was non-finite after rounding (cleared per search)  [7] an index ROW was (sticky until reset / requantise)
  int* counters = nullptr;
  uint64_t* chunk_keys = nullptr; size_t chunk_keys_elems = 0;
  // last search
  ance_search_stats stats{};
  cudaStream_t last_stream = nullptr;
};

namespace {

constexpr int kMaxPace = 256;
// k <= 512 keeps reservoirs of 1024 / 2048 (k' <= 992).  512 < k <= kMaxK takes the large-k path: reservoirs of
// kWideCap, k' in [kWideKPrimeMin, kWideKPrimeMax], at most kWideSortKeys candidates per query (the rescore sorts them in
// shared memory), queries in blocks of at most kWideQBlock so that the workspace does not grow with nq.
constexpr int kMaxK = 2048;
constexpr int kWideCap = 8192;
constexpr int kWideKPrimeMin = 1024, kWideKPrimeMax = 4096;
constexpr int kWideSortKeys = 8192;
constexpr int kWideQBlock = 16384;
constexpr int kCntQueryErr = 6, kCntRowErr = 7, kNumCounters = 8;

template <class T>
int ensure(T** ptr, size_t* have, size_t want) {
  if (*have >= want) return ANCE_OK;
  if (*ptr) cudaFree(*ptr);
  *ptr = nullptr;
  *have = 0;
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(ptr), want * sizeof(T));
  if (e != cudaSuccess) {
    ance::set_error("cudaMalloc(%zu bytes) failed: %s", want * sizeof(T), cudaGetErrorString(e));
    return ANCE_ERR_NOMEM;
  }
  *have = want;
  return ANCE_OK;
}

int check_device() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    ance::set_error("no CUDA device: %s (libance_b200 has no CPU fallback)", cudaGetErrorString(e));
    return ANCE_ERR_CUDA;
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    ance::set_error("device %d has compute capability %d.%d; libance_b200 is built for sm_90a only", dev, major, minor);
    return ANCE_ERR_CUDA;
  }
  return ANCE_OK;
}

// handles are bound to the device that was current at creation (header): refuse anything else instead of launching
// on the wrong GPU
int check_handle_device(const ance_index* ix, const char* who) {
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == ix->device, "%s: the index belongs to device %d but device %d is current", who, ix->device, dev);
  return ANCE_OK;
}

template <int BN, int STAGES, int CG, int CAP, uint32_t FMT>
int launch_coarse(ance_index* ix, const uint16_t* Q16, int64_t nq, int kprime, int out_cap, const float* thr_init,
                  int n_splits_req, int* n_splits_out, cudaStream_t st) {
  using Ep = EpTopK<BN, CAP, (CAP > 2048)>;   // CAP > 2048: EpTopKWide (streaming compaction)
  const int N = static_cast<int>(ix->n);
  gemm::WorkShape ws = gemm::make_shape(static_cast<int>(nq), N, ix->dim, BN, CG, n_splits_req);
  *n_splits_out = ws.n_splits;
  // One sweep per query tile: every concurrently running CTA pair re-reads the same corpus tile, so keep it in L2.
  // With row-range splits each pair streams its own range once: do not let it evict the (re-read) query tiles.
  ws.hint_b = (ws.n_splits == 1) ? tc05::kEvictNormal : tc05::kEvictFirst;
  CUtensorMap tmA, tmB;
  if (!tc05_host::make_tmap_2d_16b(&tmA, Q16, nq, ix->dim, ix->dim, gemm::BM) ||
      !tc05_host::make_tmap_2d_16b(&tmB, ix->P16, ix->n, ix->dim, ix->dim, BN / CG)) {
    ance::set_error("cuTensorMapEncodeTiled failed (nq=%lld n=%lld d=%d)", (long long)nq, (long long)ix->n, ix->dim);
    return ANCE_ERR_CUDA;
  }
  const int ctas = (ix->max_ctas > 0 ? ix->max_ctas : gemm::sm_count());
  size_t se = ix->scratch_elems;
  const size_t res = static_cast<size_t>(ctas) * gemm::BM * std::max(CAP, 2048);
  int rc = ensure(&ix->scratch_sc, &se, res);
  if (rc) return rc;
  se = ix->scratch_elems;
  rc = ensure(&ix->scratch_id, &se, res);
  if (rc) return rc;
  ix->scratch_elems = se;
  const size_t slots = static_cast<size_t>(nq) * ws.n_splits;
  size_t a = ix->cand_slots, b = ix->cand_slots;
  if ((rc = ensure(&ix->cand_cnt, &a, slots))) return rc;
  if ((rc = ensure(&ix->cand_thr, &b, slots))) return rc;
  ix->cand_slots = a;
  if ((rc = ensure(&ix->cand_id, &ix->cand_ids, slots * out_cap))) return rc;
  // Soft barrier between the sweeping CTA pairs (gemm_core.cuh): pairs that sweep the SAME corpus rows share each tile
  // through L2 as long as they stay within `pace_window` tiles of each other.  Without it they drift apart and every one of
  // them streams the rows from HBM by itself.  Two shapes qualify: every item sweeps the whole
  // corpus (n_splits == 1: all pairs pace each other), or one wave of (query tile, row range) items (pairs with the same
  // range pace each other).
  const int total_items = ws.num_m_blks * ws.n_splits;
  const int clusters = std::min(total_items, ctas / CG);
  const bool whole = ws.n_splits == 1 && clusters > 1;
  const bool one_wave = ws.n_splits > 1 && ws.num_m_blks > 1 && total_items <= ctas / CG;
  if ((whole || one_wave) && clusters <= kMaxPace && ix->pace_window > 0 && ws.n_blks_per_split > 4 * ix->pace_window) {
    ANCE_CUDA(cudaMemsetAsync(ix->pace, 0, kMaxPace * sizeof(int), st));
    ws.pace = ix->pace;
    ws.pace_window = ix->pace_window;
    ws.pace_stride = whole ? 1 : ws.n_splits;
    ws.hint_b = tc05::kEvictNormal;   // the tile is re-read by the other pairs of the group: keep it in L2
  }
  typename Ep::Params p;
  p.scratch_sc = ix->scratch_sc;
  p.scratch_id = ix->scratch_id;
  p.cand_id = ix->cand_id;
  p.cand_cnt = ix->cand_cnt;
  p.cand_thr = ix->cand_thr;
  p.thr_init = thr_init;
  p.kprime = kprime;
  p.out_cap = out_cap;
  p.nq = static_cast<int>(nq);
  p.n_rows = N;
  {
    ance::ProfScope ps(ance::kClsCoarse, st);
    ANCE_CUDA((gemm::launch<Ep, BN, STAGES, CG, 4, FMT>(tmA, tmB, ws, p, ctas, st)));
  }
  ance::count_launch(1);
  return ANCE_OK;
}

constexpr int kExactBatch = 1024;  // queries per brute-force pass (bounds the chunk_keys scratch)
// k > 512: fewer queries per pass, so that chunk_keys (batch * n_chunks * k * 8 bytes) stays within this
constexpr size_t kExactKeysBytes = size_t(512) << 20;

// device staging buffer of a host index's prepare and brute force
constexpr size_t kHostStageBytes = size_t(512) << 20;

// run_exact on a host index: the rows cross PCIe ONCE per batch of queries.  For each batch the rows are copied H2D slab by
// slab (at most 512 MB) into a staging buffer; the device brute force runs on the slab with global row numbers and keeps
// its chunk keys next to a per-query slot holding the best k of the earlier slabs, which exact_merge_kernel<true> updates
// after every slab; after the last slab exact_merge_kernel<false> writes D / I.  The result is the device path's: the
// same keys (score, then global row) merged by the same kernels.
int run_exact_host(ance_index* ix, const float* Q, const int* qlist, int nq, int k, float* D, int64_t* I,
                   int64_t row_offset, cudaStream_t st) {
  const int d = ix->dim;
  const int64_t n = ix->n;
  const int64_t slab = std::min<int64_t>(n, std::max<int64_t>(1, static_cast<int64_t>(kHostStageBytes / (static_cast<size_t>(d) * 4))));
  ExactParams ep;
  ep.Q = Q;
  ep.d = d;
  ep.nq_dev = nullptr;
  ep.k = static_cast<int>(std::min<int64_t>(std::min<int64_t>(k, std::max<int64_t>(n, 1)), kMaxK));
  const int sms = gemm::sm_count();
  const int n_chunks = std::max(1, static_cast<int>(std::min<int64_t>(2 * sms, (slab + 4095) / 4096)));
  ep.n_chunks = n_chunks;
  const bool large = ep.k > 512;
  const size_t per_query = static_cast<size_t>(n_chunks + 1) * ep.k * 8;
  int batch = std::min(nq, kExactBatch);
  if (large) batch = std::min<int>(batch, std::max<int>(kExQB, static_cast<int>(kExactKeysBytes / per_query) / kExQB * kExQB));
  int rc = ensure(&ix->chunk_keys, &ix->chunk_keys_elems, static_cast<size_t>(batch) * (n_chunks + 1) * ep.k);
  if (rc) return rc;
  ep.chunk_keys = ix->chunk_keys;
  const int buf = large ? kExBufLarge : kExBufSmall;
  const size_t smem = static_cast<size_t>(kExQB) * buf * 8 + static_cast<size_t>(kExQB) * d * 4;
  auto chunk_kernel = large ? exact_chunk_kernel<kExBufLarge, true> : exact_chunk_kernel<kExBufSmall, true>;
  ANCE_CUDA(cudaFuncSetAttribute(chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 large ? static_cast<int>(smem) : 100 * 1024));
  float* stage = nullptr;
  cudaError_t e = cudaMalloc(&stage, static_cast<size_t>(slab) * d * 4);
  if (e != cudaSuccess) {
    ance::set_error("ance_index_search_exact: cudaMalloc(%lld bytes) of the staging buffer failed: %s",
                    (long long)(slab * d * 4), cudaGetErrorString(e));
    return ANCE_ERR_NOMEM;
  }
  for (int b0 = 0; b0 < nq && e == cudaSuccess; b0 += batch) {
    const int nb = std::min(batch, nq - b0);
    ep.qlist = qlist ? qlist + b0 : nullptr;
    ep.q_base = b0;
    ep.nq = nb;
    const int gy = std::max(1, std::min((nb + kExQB - 1) / kExQB, 128));
    ance::ProfScope ps(ance::kClsExact, st);
    e = cudaMemsetAsync(ep.chunk_keys, 0, static_cast<size_t>(nb) * (n_chunks + 1) * ep.k * 8, st);   // empty best-k slots
    for (int64_t r0 = 0; r0 < n && e == cudaSuccess; r0 += slab) {
      const int64_t m = std::min(slab, n - r0);
      e = cudaMemcpyAsync(stage, ix->P32_host + r0 * d, static_cast<size_t>(m) * d * 4, cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) break;
      ep.P = stage;
      ep.n_rows = m;
      chunk_kernel<<<dim3(n_chunks, gy), 256, smem, st>>>(ep, r0);
      ExactParams mp = ep;
      mp.n_chunks = n_chunks + 1;   // the chunk keys and the running best-k slot
      if (r0 + m < n)
        exact_merge_kernel<true><<<std::max(1, std::min(nb, 4 * sms)), 256, 0, st>>>(mp, nullptr, nullptr, k, row_offset);
      else
        exact_merge_kernel<false><<<std::max(1, std::min(nb, 4 * sms)), 256, 0, st>>>(mp, D, I, k, row_offset);
      ance::count_launch(2);
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // the staging buffer is in use until here
  cudaFree(stage);
  if (e != cudaSuccess) {
    ance::set_error("ance_index_search_exact (host rows): %s", cudaGetErrorString(e));
    return ANCE_ERR_CUDA;
  }
  return ANCE_OK;
}

int run_exact(ance_index* ix, const float* Q, const int* qlist, int nq, int k, float* D, int64_t* I,
              int64_t row_offset, cudaStream_t st) {
  if (ix->host_rows) return run_exact_host(ix, Q, qlist, nq, k, D, I, row_offset, st);
  ExactParams ep;
  ep.Q = Q;
  ep.P = ix->P32;
  ep.d = ix->dim;
  ep.n_rows = ix->n;
  ep.nq_dev = nullptr;
  ep.k = static_cast<int>(std::min<int64_t>(k, std::max<int64_t>(ix->n, 1)));
  ep.k = std::min(ep.k, kMaxK);
  const int sms = gemm::sm_count();
  int n_chunks = static_cast<int>(std::min<int64_t>(2 * sms, (ix->n + 4095) / 4096));
  if (n_chunks < 1) n_chunks = 1;
  ep.n_chunks = n_chunks;
  const bool large = ep.k > 512;
  int batch = std::min(nq, kExactBatch);
  if (large) {
    const size_t per_query = static_cast<size_t>(n_chunks) * ep.k * 8;
    batch = std::min<int>(batch, std::max<int>(kExQB, static_cast<int>(kExactKeysBytes / per_query) / kExQB * kExQB));
  }
  int rc = ensure(&ix->chunk_keys, &ix->chunk_keys_elems, static_cast<size_t>(batch) * n_chunks * ep.k);
  if (rc) return rc;
  ep.chunk_keys = ix->chunk_keys;
  const int buf = large ? kExBufLarge : kExBufSmall;
  const size_t smem = static_cast<size_t>(kExQB) * buf * 8 + static_cast<size_t>(kExQB) * ix->dim * 4;
  // per device and cheap: set on every call rather than behind a process-wide flag
  auto chunk_kernel = large ? exact_chunk_kernel<kExBufLarge, false> : exact_chunk_kernel<kExBufSmall, false>;
  ANCE_CUDA(cudaFuncSetAttribute(chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 large ? static_cast<int>(smem) : 100 * 1024));
  for (int b0 = 0; b0 < nq; b0 += batch) {
    const int nb = std::min(batch, nq - b0);
    ep.qlist = qlist ? qlist + b0 : nullptr;
    ep.q_base = b0;
    ep.nq = nb;
    const int gy = std::max(1, std::min((nb + kExQB - 1) / kExQB, 128));
    ance::ProfScope ps(ance::kClsExact, st);
    chunk_kernel<<<dim3(n_chunks, gy), 256, smem, st>>>(ep, 0);
    ANCE_CUDA(cudaGetLastError());
    exact_merge_kernel<false><<<std::max(1, std::min(nb, 4 * sms)), 256, 0, st>>>(ep, D, I, k, row_offset);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(2);
  }
  return ANCE_OK;
}

// One coarse pass + exact rescoring + certificate over `nq` queries whose 16-bit rows are Q16[0..nq);
// qlist (or identity) maps them to rows of q_f32 / D / I.  thr_init == null: tier 1 (running top-k' from -inf, k'
// candidates per split kept).  thr_init != null: tier 2 (start from the per-query threshold, keep everything that
// passes it).  Uncertified queries are appended to flagged_out (+ their next-tier threshold to flagged_thr_out) and
// counted in counters[flag_slot].
int coarse_rescore_pass(ance_index* ix, const uint16_t* Q16, const float* q_f32, int64_t nq, const int* qlist,
                        int kprime, const float* thr_init, int n_splits_req, int k, float* D_dev, int64_t* I_dev,
                        int64_t row_offset, int* flagged_out, float* flagged_thr_out, int flag_slot, int* ns_out,
                        cudaStream_t st) {
  int rc;
  const int cap = (kprime <= 512) ? 1024 : (kprime <= 992) ? 2048 : kWideCap;
  // candidates per query that rescore_kernel sorts in shared memory
  const int max_keys = (cap == kWideCap) ? kWideSortKeys : 4096;
  // tier 2 keeps whatever the reservoir holds at the end (at most cap - 32 entries: a fuller one is compacted at once)
  const int out_cap = thr_init ? cap : kprime;
  const int cg = ix->cta_group;
  const int clusters = (ix->max_ctas > 0 ? ix->max_ctas : gemm::sm_count()) / cg;
  const int q_tiles = static_cast<int>((nq + gemm::BM * cg - 1) / (gemm::BM * cg));
  int n_splits = n_splits_req;
  if (n_splits == 0) {
    // Few query tiles: split the corpus into row ranges so that every CTA (pair) has work, choosing the
    // split count whose work-item count fills whole waves best (ties: fewer splits = fewer candidates).
    n_splits = 1;
    if (q_tiles < 2 * clusters) {
      const int max_splits = std::max(1, std::min(16, max_keys / out_cap));
      double best = -1.0;
      for (int sp = 1; sp <= max_splits; ++sp) {
        const long items = static_cast<long>(q_tiles) * sp;
        const long waves = (items + clusters - 1) / clusters;
        const double eff = static_cast<double>(items) / static_cast<double>(waves * clusters);
        if (eff > best + 1e-9) { best = eff; n_splits = sp; }
      }
    }
  }
  while (n_splits > 1 && n_splits * out_cap > max_keys) --n_splits;
  ANCE_REQUIRE(n_splits * out_cap <= max_keys, "ance_index_search: n_splits * candidates per split = %d exceeds %d",
               n_splits * out_cap, max_keys);
  int ns = 0;
  const bool bf = ix->fmt == ANCE_FMT_BF16;
#define ANCE_COARSE(CG_, CAP_)                                                                                              \
  rc = bf ? launch_coarse<128, 4, CG_, CAP_, tc05::kFmtBF16>(ix, Q16, nq, kprime, out_cap, thr_init, n_splits, &ns, st) \
          : launch_coarse<128, 4, CG_, CAP_, tc05::kFmtF16>(ix, Q16, nq, kprime, out_cap, thr_init, n_splits, &ns, st)
  if (cap == kWideCap) {
    if (cg == 1) { ANCE_COARSE(1, kWideCap); }
    else { ANCE_COARSE(2, kWideCap); }
  }
  else if (cg == 1 && cap == 1024) { ANCE_COARSE(1, 1024); }
  else if (cg == 1) { ANCE_COARSE(1, 2048); }
  else if (cap == 1024) { ANCE_COARSE(2, 1024); }
  else { ANCE_COARSE(2, 2048); }
#undef ANCE_COARSE
  if (rc) return rc;
  *ns_out = ns;
  RescoreParams rp;
  rp.Q = q_f32;
  rp.P = ix->P32;
  rp.d = ix->dim;
  rp.cand_id = ix->cand_id;
  rp.cand_cnt = ix->cand_cnt;
  rp.cand_thr = ix->cand_thr;
  rp.n_splits = ns;
  rp.cand_stride = out_cap;
  rp.k = k;
  rp.qn_hat = ix->qn_hat;
  rp.qn_delta = ix->qn_delta;
  rp.pstats = ix->pstats;
  rp.mu = ix->centred ? ix->mu : nullptr;
  // Accumulation error of the coarse score c = fl(sum_i q^_i p^_i) on the tensor core.  The 16-bit x 16-bit products
  // are exact in fp32; what is unspecified is how wgmma adds them (PTX: "precision at least that of fp32", order
  // and rounding implementation-defined; published measurements of earlier generations: truncation, block adds of
  // K = 16 aligned to the largest exponent).  Any such scheme performs at most d + d/16 additions, each with an error
  // of at most one ulp of the largest partial sum, 2^-23 * sum_i |q^_i p^_i| <= 2^-23 ||q^|| ||p^|| (Cauchy-Schwarz):
  //   |c - <q^, p^>| <= (17/16) d 2^-23 ||q^|| ||p^||  <  d * 2^-22 * ||q^|| ||p^||          (d = 768: 1.83e-4)
  // tests/test_gpu_search.py measures the real error against an fp64 dot of the same rounded operands (it is ~300x
  // smaller: rounding errors average out, the bound does not assume they do).
  rp.accum_rel = static_cast<float>(ix->dim) * 2.384185791015625e-07f;
  rp.D = D_dev;
  rp.I = I_dev;
  rp.row_offset = row_offset;
  rp.qlist = qlist;
  rp.flagged_list = flagged_out;
  rp.flagged_thr = flagged_thr_out;
  rp.flag_slot = flag_slot;
  rp.counters = ix->counters;
  rp.max_eps = reinterpret_cast<unsigned int*>(ix->counters + 2);
  rp.sort_n = next_pow2(ns * out_cap);
  rp.P16 = ix->P16;
  rp.ndelta = ix->ndelta;
  rp.bf16 = bf;
  size_t rs_smem = static_cast<size_t>(rp.sort_n) * 8 + static_cast<size_t>(ix->dim) * 4 + (ns + 1) * 4 + 16;
  // host index: + per-candidate upper bounds (fp64), rows and survivors after the 16-byte aligned base layout
  // (8192 candidates: 64 KB keys + 128 KB = 195 KB at d = 768)
  if (ix->host_rows) rs_smem = ((rs_smem - 16 + 15) & ~size_t(15)) + static_cast<size_t>(rp.sort_n) * 16;
  auto kern = ix->host_rows ? rescore_kernel<true> : rescore_kernel<false>;
  if (rs_smem > 48 * 1024)   // per device and cheap: no process-wide cache
    ANCE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rs_smem)));
  ance::prof_begin(ance::kClsRescore, st);
  kern<<<static_cast<unsigned>(nq), 256, rs_smem, st>>>(rp);
  ance::prof_end(ance::kClsRescore, st);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

// host_rows: the fp32 rows live in pinned host memory (external_rows = caller-owned page-locked buffer, or null: allocated
// here); otherwise external_rows is caller-owned device storage, or null: allocated here.
int create_common(int dim, int64_t capacity_rows, int operand_fmt, float* external_rows, bool host_rows, ance_index_t* out) {
  ANCE_REQUIRE(out != nullptr, "ance_index_create: out is null");
  ANCE_REQUIRE(dim > 0 && dim % 8 == 0 && dim <= 4096, "ance_index_create: dim must be a multiple of 8 in (0, 4096], got %d", dim);
  ANCE_REQUIRE(capacity_rows > 0 && capacity_rows < (1ll << 31), "ance_index_create: capacity_rows out of range");
  ANCE_REQUIRE(operand_fmt == ANCE_FMT_BF16 || operand_fmt == ANCE_FMT_FP16, "ance_index_create: bad operand_fmt");
  int rc = check_device();
  if (rc) return rc;
  float* host_dev = nullptr;   // device address of caller-owned host rows
  if (host_rows && external_rows) {
    cudaPointerAttributes a{};
    const cudaError_t e = cudaPointerGetAttributes(&a, external_rows);
    if (e != cudaSuccess) cudaGetLastError();   // not a sticky error: clear it
    ANCE_REQUIRE(e == cudaSuccess && a.type == cudaMemoryTypeHost && a.devicePointer != nullptr &&
                 (reinterpret_cast<uintptr_t>(external_rows) & 15) == 0,
                 "ance_index_create_host: rows_host must be 16-byte aligned page-locked host memory mapped into the device");
    host_dev = static_cast<float*>(a.devicePointer);
  }
  ance_index* ix = new ance_index();
  ix->dim = dim;
  ix->cap = capacity_rows;
  ix->fmt = operand_fmt;
  ix->host_rows = host_rows;
  cudaGetDevice(&ix->device);
  const size_t elems = static_cast<size_t>(capacity_rows) * dim;
  cudaError_t e1 = cudaSuccess;
  if (host_rows) {
    ix->owns_p32 = false;
    if (external_rows) {
      ix->P32_host = external_rows;
      ix->P32 = host_dev;
    } else {
      e1 = cudaHostAlloc(reinterpret_cast<void**>(&ix->P32_host), elems * 4, cudaHostAllocMapped | cudaHostAllocPortable);
      if (e1 == cudaSuccess) {
        ix->owns_host = true;
        e1 = cudaHostGetDevicePointer(reinterpret_cast<void**>(&ix->P32), ix->P32_host, 0);
      }
    }
    if (e1 == cudaSuccess) e1 = cudaMalloc(&ix->ndelta, static_cast<size_t>(capacity_rows) * sizeof(float));
  } else if (external_rows) {
    ix->P32 = external_rows;
    ix->owns_p32 = false;
  } else {
    e1 = cudaMalloc(&ix->P32, elems * 4);
  }
  cudaError_t e2 = cudaMalloc(&ix->P16, elems * 2);
  cudaError_t e3 = cudaMalloc(&ix->pstats, 2 * sizeof(unsigned int));
  cudaError_t e4 = cudaMalloc(&ix->pace, kMaxPace * sizeof(int));
  cudaError_t e5 = cudaMalloc(&ix->counters, kNumCounters * sizeof(int));
  cudaError_t e6 = cudaMalloc(&ix->mu, static_cast<size_t>(dim) * sizeof(float));
  cudaError_t e7 = cudaMalloc(&ix->colsum, static_cast<size_t>(dim) * sizeof(double));
  if (e1 || e2 || e3 || e4 || e5 || e6 || e7) {
    ance::set_error("ance_index_create%s: %s failed for %lld x %d rows", host_rows ? "_host" : "",
                    host_rows ? "cudaHostAlloc / cudaMalloc" : "cudaMalloc", (long long)capacity_rows, dim);
    ance_index_destroy(ix);
    return ANCE_ERR_NOMEM;
  }
  cudaMemset(ix->pstats, 0, 2 * sizeof(unsigned int));
  cudaMemset(ix->counters, 0, kNumCounters * sizeof(int));
  *out = ix;
  return ANCE_OK;
}

// prepare_operands of a host index: the fp32 rows are streamed H2D in chunks through a staging buffer of at most 512 MB
// (one pass for the column sums when centring, one for the rounding), and the same kernels as the device index's run on
// each chunk.  The rounding also stores every row's ||delta_j|| (ndelta), which the rescoring pre-filter needs.  The
// staging buffer is freed at the end: the index keeps 2 bytes per row element + 4 bytes per row on the device.
int prepare_operands_host(ance_index* ix, cudaStream_t st) {
  const int64_t n = ix->n;
  if (n == 0) return ANCE_OK;
  const int d = ix->dim;
  const int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(1, static_cast<int64_t>(kHostStageBytes / (static_cast<size_t>(d) * 4))));
  float* stage = nullptr;
  cudaError_t e = cudaMalloc(&stage, static_cast<size_t>(chunk) * d * 4);
  if (e != cudaSuccess) {
    ance::set_error("ance_index_prepare: cudaMalloc(%lld bytes) of the staging buffer failed: %s",
                    (long long)(chunk * d * 4), cudaGetErrorString(e));
    return ANCE_ERR_NOMEM;
  }
  auto stream_pass = [&](bool quantize) -> cudaError_t {
    for (int64_t r0 = 0; r0 < n; r0 += chunk) {
      const int64_t m = std::min(chunk, n - r0);
      cudaError_t err = cudaMemcpyAsync(stage, ix->P32_host + r0 * d, static_cast<size_t>(m) * d * 4, cudaMemcpyHostToDevice, st);
      if (err != cudaSuccess) return err;
      if (!quantize) {
        const int slab = static_cast<int>(std::min<int64_t>(4096, std::max<int64_t>(32, m / (8 * gemm::sm_count()))));
        column_sum_kernel<<<static_cast<unsigned>((m + slab - 1) / slab), 256, 0, st>>>(stage, m, d, slab, ix->colsum);
      } else {
        const float* mu = ix->centred ? ix->mu : nullptr;
        const unsigned blocks = static_cast<unsigned>((m + 7) / 8);
        uint16_t* o16 = ix->P16 + r0 * d;
        if (ix->fmt == ANCE_FMT_BF16)
          quantize_rows_kernel<true><<<blocks, 256, 0, st>>>(stage, o16, m, d, mu, nullptr, ix->ndelta + r0, ix->pstats, ix->counters + kCntRowErr);
        else
          quantize_rows_kernel<false><<<blocks, 256, 0, st>>>(stage, o16, m, d, mu, nullptr, ix->ndelta + r0, ix->pstats, ix->counters + kCntRowErr);
      }
      ance::count_launch(1);
      if ((err = cudaGetLastError()) != cudaSuccess) return err;
    }
    return cudaSuccess;
  };
  if (ix->centred) {
    e = cudaMemsetAsync(ix->colsum, 0, static_cast<size_t>(d) * sizeof(double), st);
    if (e == cudaSuccess) e = stream_pass(false);
    if (e == cudaSuccess) {
      finalize_mean_kernel<<<(d + 255) / 256, 256, 0, st>>>(ix->colsum, n, d, ix->mu);
      ance::count_launch(1);
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) e = stream_pass(true);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // the staging buffer is in use until here
  cudaFree(stage);
  if (e != cudaSuccess) {
    ance::set_error("ance_index_prepare (host rows): %s", cudaGetErrorString(e));
    return ANCE_ERR_CUDA;
  }
  return ANCE_OK;
}

// (Re)build the 16-bit operands of every row from the fp32 rows: column mean -> centre -> round, norm maxima, range flag.
// Runs once per index state (lazily, at the first search after rows were added): ~45 GB of HBM traffic for 8.84M rows,
// about 10 ms — nothing next to the encode that produced the rows — and it lets the centre be the mean of ALL rows.
int prepare_operands(ance_index* ix, cudaStream_t st) {
  if (!ix->dirty) return ANCE_OK;
  const int64_t n = ix->n;
  ANCE_CUDA(cudaMemsetAsync(ix->pstats, 0, 2 * sizeof(unsigned int), st));
  ANCE_CUDA(cudaMemsetAsync(ix->counters + kCntRowErr, 0, sizeof(int), st));
  ance::ProfScope ps(ance::kClsQuant, st);
  ix->centred = ix->center && n >= 256;
  if (ix->host_rows) {
    int rc = prepare_operands_host(ix, st);
    if (rc) return rc;
    ix->dirty = false;
    return ANCE_OK;
  }
  if (ix->centred) {
    ANCE_CUDA(cudaMemsetAsync(ix->colsum, 0, static_cast<size_t>(ix->dim) * sizeof(double), st));
    // rows per block: enough blocks to fill the machine for a small index, few enough atomics (n / slab per column) for a big one
    const int slab = static_cast<int>(std::min<int64_t>(4096, std::max<int64_t>(32, n / (8 * gemm::sm_count()))));
    column_sum_kernel<<<static_cast<unsigned>((n + slab - 1) / slab), 256, 0, st>>>(ix->P32, n, ix->dim, slab, ix->colsum);
    finalize_mean_kernel<<<(ix->dim + 255) / 256, 256, 0, st>>>(ix->colsum, n, ix->dim, ix->mu);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(2);
  }
  const float* mu = ix->centred ? ix->mu : nullptr;
  const int wpb = 8;
  const unsigned blocks = static_cast<unsigned>((n + wpb - 1) / wpb);
  if (n > 0) {
    if (ix->fmt == ANCE_FMT_BF16)
      quantize_rows_kernel<true><<<blocks, wpb * 32, 0, st>>>(ix->P32, ix->P16, n, ix->dim, mu, nullptr, nullptr, ix->pstats, ix->counters + kCntRowErr);
    else
      quantize_rows_kernel<false><<<blocks, wpb * 32, 0, st>>>(ix->P32, ix->P16, n, ix->dim, mu, nullptr, nullptr, ix->pstats, ix->counters + kCntRowErr);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
  }
  ix->dirty = false;
  return ANCE_OK;
}

// Tiers 1-3 of one search over queries q_dev[0, nq) into D / I [nq, k]; the counts are added to *acc (nq, kprime and
// the stream are the caller's).  tier2_kprime: what tier 2 compacts an overflowing reservoir to (>= k).
int search_tiers(ance_index* ix, const float* q_dev, int64_t nq, int k, int kprime, int tier2_kprime, float* D_dev,
                 int64_t* I_dev, int64_t row_offset, cudaStream_t st, ance_search_stats* acc) {
  int rc;
  // --- 1. quantize queries
  {
    size_t a = static_cast<size_t>(ix->q_cap) * ix->dim, b = ix->q_cap, c = ix->q_cap;
    if ((rc = ensure(&ix->Q16, &a, static_cast<size_t>(nq) * ix->dim))) return rc;
    if ((rc = ensure(&ix->qn_hat, &b, static_cast<size_t>(nq)))) return rc;
    if ((rc = ensure(&ix->qn_delta, &c, static_cast<size_t>(nq)))) return rc;
    ix->q_cap = std::max<int64_t>(ix->q_cap, nq);
    size_t f = ix->flagged_cap, g = ix->flagged_cap;
    if ((rc = ensure(&ix->flagged, &f, static_cast<size_t>(nq)))) return rc;
    if ((rc = ensure(&ix->flagged_thr, &g, static_cast<size_t>(nq)))) return rc;
    ix->flagged_cap = f;
  }
  ANCE_CUDA(cudaMemsetAsync(ix->counters, 0, kCntRowErr * sizeof(int), st));   // everything but the sticky row flag
  const unsigned qblocks = static_cast<unsigned>((nq + 7) / 8);
  ance::prof_begin(ance::kClsQuant, st);
  if (ix->fmt == ANCE_FMT_BF16)
    quantize_rows_kernel<true><<<qblocks, 256, 0, st>>>(q_dev, ix->Q16, nq, ix->dim, nullptr, ix->qn_hat, ix->qn_delta, nullptr, ix->counters + kCntQueryErr);
  else
    quantize_rows_kernel<false><<<qblocks, 256, 0, st>>>(q_dev, ix->Q16, nq, ix->dim, nullptr, ix->qn_hat, ix->qn_delta, nullptr, ix->counters + kCntQueryErr);
  ance::prof_end(ance::kClsQuant, st);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  // --- 2+3. tier 1: coarse pass over all queries, exact rescoring, certificate
  int ns = 0;
  rc = coarse_rescore_pass(ix, ix->Q16, q_dev, nq, nullptr, kprime, nullptr, ix->n_splits, k, D_dev, I_dev, row_offset,
                           ix->flagged, ix->flagged_thr, 0, &ns, st);
  if (rc) return rc;
  // One small D2H + sync per search tells the host how many queries stay uncertified and whether an operand left
  // the 16-bit format's range (the reference's search call is synchronous as well).
  int h[kNumCounters] = {};
  ANCE_CUDA(cudaMemcpyAsync(h, ix->counters, sizeof(h), cudaMemcpyDeviceToHost, st));
  ANCE_CUDA(cudaStreamSynchronize(st));
  if (h[kCntQueryErr] || h[kCntRowErr]) {
    // coarse scores, thresholds and the certificate would be compared against inf / NaN: refuse instead of
    // returning ANCE_OK with unverifiable neighbours
    ance::set_error("ance_index_search: %s non-finite after rounding to %s (inf / NaN in the input%s)",
                    h[kCntRowErr] ? "an index row is" : "a query is", ix->fmt == ANCE_FMT_FP16 ? "fp16" : "bf16",
                    ix->fmt == ANCE_FMT_FP16 ? ", or |x| > 65504: switch with ance_index_set_param(\"operand_fmt\", ANCE_FMT_BF16)" : "");
    return ANCE_ERR_UNSUPPORTED;
  }
  int n_exact = h[0];
  int ns2 = 0;
  if (h[0] > 0 && ix->tier2 && ix->n >= 4 * static_cast<int64_t>(tier2_kprime)) {
    // --- tier 2: the uncertified queries once more, from their own thresholds (nothing that passes is dropped)
    const int n2 = h[0];
    if ((rc = ensure(&ix->Q16b, &ix->q16b_elems, static_cast<size_t>(n2) * ix->dim))) return rc;
    if ((rc = ensure(&ix->flagged2, &ix->flagged2_cap, static_cast<size_t>(n2)))) return rc;
    gather_rows16_kernel<<<n2, 96, 0, st>>>(ix->Q16, ix->flagged, n2, ix->dim, ix->Q16b);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
    rc = coarse_rescore_pass(ix, ix->Q16b, q_dev, n2, ix->flagged, tier2_kprime, ix->flagged_thr, 0, k, D_dev, I_dev, row_offset,
                             ix->flagged2, nullptr, 3, &ns2, st);
    if (rc) return rc;
    ANCE_CUDA(cudaMemcpyAsync(h, ix->counters, sizeof(h), cudaMemcpyDeviceToHost, st));
    ANCE_CUDA(cudaStreamSynchronize(st));
    n_exact = h[3];
    if (n_exact > 0 && ix->exact_fallback) {
      rc = run_exact(ix, q_dev, ix->flagged2, n_exact, k, D_dev, I_dev, row_offset, st);
      if (rc) return rc;
    }
  } else if (n_exact > 0 && ix->exact_fallback) {
    // --- tier 3: exact brute force
    rc = run_exact(ix, q_dev, ix->flagged, n_exact, k, D_dev, I_dev, row_offset, st);
    if (rc) return rc;
  }
  ix->last_fetched += h[kCntFetched];   // tiers 1 and 2 (the counters are cleared once per block, above)
  acc->n_splits = std::max(acc->n_splits, ns);
  acc->n_tier2 += h[0];
  acc->n_uncertified += n_exact;
  acc->n_candidates += h[1];
  float eps;
  memcpy(&eps, &h[2], 4);
  acc->max_eps = std::max(acc->max_eps, eps);
  return ANCE_OK;
}

}  // namespace

extern "C" int ance_index_create(int dim, int64_t capacity_rows, int operand_fmt, ance_index_t* out) {
  return create_common(dim, capacity_rows, operand_fmt, nullptr, false, out);
}

extern "C" int ance_index_create_host(int dim, int64_t capacity_rows, int operand_fmt, float* rows_host, ance_index_t* out) {
  return create_common(dim, capacity_rows, operand_fmt, rows_host, true, out);
}

extern "C" int ance_index_create_over(int dim, int64_t capacity_rows, int operand_fmt, float* rows_dev,
                                      ance_index_t* out) {
  ANCE_REQUIRE(rows_dev != nullptr, "ance_index_create_over: rows_dev is null");
  ANCE_REQUIRE((reinterpret_cast<uintptr_t>(rows_dev) & 15) == 0, "ance_index_create_over: rows_dev must be 16-byte aligned");
  return create_common(dim, capacity_rows, operand_fmt, rows_dev, false, out);
}

extern "C" int ance_index_destroy(ance_index_t ix) {
  if (!ix) return ANCE_OK;
  void* ptrs[] = {ix->owns_p32 ? ix->P32 : nullptr, ix->P16, ix->pstats, ix->Q16, ix->qn_hat, ix->qn_delta, ix->scratch_sc,
                  ix->scratch_id, ix->cand_id, ix->cand_cnt, ix->cand_thr, ix->flagged, ix->flagged_thr, ix->counters,
                  ix->chunk_keys, ix->flagged2, ix->Q16b, ix->pace, ix->mu, ix->colsum, ix->ndelta};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  if (ix->owns_host) cudaFreeHost(ix->P32_host);
  delete ix;
  return ANCE_OK;
}

extern "C" int ance_index_reset(ance_index_t ix) {
  ANCE_REQUIRE(ix != nullptr, "ance_index_reset: null handle");
  ix->n = 0;
  ix->dirty = false;
  ANCE_CUDA(cudaMemset(ix->pstats, 0, 2 * sizeof(unsigned int)));
  ANCE_CUDA(cudaMemset(ix->counters, 0, kNumCounters * sizeof(int)));
  return ANCE_OK;
}

extern "C" int64_t ance_index_ntotal(ance_index_t ix) { return ix ? ix->n : -1; }

extern "C" int ance_index_add(ance_index_t ix, const float* rows_dev, int64_t n, void* stream) {
  ANCE_REQUIRE(ix != nullptr, "ance_index_add: null handle");
  ANCE_REQUIRE(n >= 0, "ance_index_add: negative row count");
  if (n == 0) return ANCE_OK;
  ANCE_REQUIRE(rows_dev != nullptr, "ance_index_add: rows_dev is null");
  ANCE_REQUIRE(ix->n + n <= ix->cap, "ance_index_add: %lld + %lld rows exceed capacity %lld", (long long)ix->n,
               (long long)n, (long long)ix->cap);
  int rc = check_handle_device(ix, "ance_index_add");
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* dst = ix->P32 + static_cast<size_t>(ix->n) * ix->dim;
  if (ix->host_rows) {
    // device rows: stream-ordered D2H into the pinned storage; any other host pointer: a plain (synchronous) copy; the
    // storage slice itself (host or device address): no copy
    float* dst_host = ix->P32_host + static_cast<size_t>(ix->n) * ix->dim;
    if (dst_host != rows_dev && dst != rows_dev)
      ANCE_CUDA(cudaMemcpyAsync(dst_host, rows_dev, static_cast<size_t>(n) * ix->dim * 4, cudaMemcpyDefault, st));
  } else if (dst != rows_dev)   // rows produced in place (the encoder wrote straight into the index storage): no copy
    ANCE_CUDA(cudaMemcpyAsync(dst, rows_dev, static_cast<size_t>(n) * ix->dim * 4, cudaMemcpyDeviceToDevice, st));
  ix->n += n;
  ix->dirty = true;      // the 16-bit operands are (re)built from all rows by the next ance_index_prepare / search
  return ANCE_OK;
}

extern "C" int ance_index_prepare(ance_index_t ix, void* stream) {
  ANCE_REQUIRE(ix != nullptr, "ance_index_prepare: null handle");
  int rc = check_handle_device(ix, "ance_index_prepare");
  if (rc) return rc;
  return prepare_operands(ix, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ance_index_set_param(ance_index_t ix, const char* name, double value) {
  ANCE_REQUIRE(ix != nullptr && name != nullptr, "ance_index_set_param: null argument");
  const int v = static_cast<int>(value);
  if (!strcmp(name, "kprime")) { ANCE_REQUIRE(v >= 0 && v <= kWideKPrimeMax && v % 32 == 0, "kprime must be a multiple of 32 in [0, %d]", kWideKPrimeMax); ix->kprime = v; }
  else if (!strcmp(name, "n_splits")) { ANCE_REQUIRE(v >= 0 && v <= 64, "n_splits must be in [0, 64]"); ix->n_splits = v; }
  else if (!strcmp(name, "cta_group")) { ANCE_REQUIRE(v == 1 || v == 2, "cta_group must be 1 or 2"); ix->cta_group = v; }
  else if (!strcmp(name, "exact_fallback")) { ix->exact_fallback = v != 0; }
  else if (!strcmp(name, "tier2")) { ix->tier2 = v != 0; }
  else if (!strcmp(name, "max_ctas")) { ANCE_REQUIRE(v >= 0, "max_ctas must be >= 0"); ix->max_ctas = v; }
  else if (!strcmp(name, "pace_window")) { ANCE_REQUIRE(v >= 0 && v <= 4096, "pace_window must be in [0, 4096]"); ix->pace_window = v; }
  else if (!strcmp(name, "operand_fmt")) {
    // re-round the rows already in the index to the other 16-bit format (the fp32 rows are kept for exactly this)
    ANCE_REQUIRE(v == ANCE_FMT_BF16 || v == ANCE_FMT_FP16, "operand_fmt must be ANCE_FMT_FP16 or ANCE_FMT_BF16");
    int rc = check_handle_device(ix, "ance_index_set_param");
    if (rc) return rc;
    if (v != ix->fmt) {
      ix->fmt = v;
      ix->dirty = true;
    }
  }
  else if (!strcmp(name, "center")) { ix->center = v != 0; ix->dirty = true; }
  else { ance::set_error("ance_index_set_param: unknown parameter '%s'", name); return ANCE_ERR_INVALID; }
  return ANCE_OK;
}

extern "C" int ance_index_search_exact(ance_index_t ix, const float* q_dev, int64_t nq, int k, float* D_dev,
                                       int64_t* I_dev, int64_t row_offset, void* stream) {
  ANCE_REQUIRE(ix != nullptr, "ance_index_search_exact: null handle");
  ANCE_REQUIRE(nq >= 0 && k > 0 && k <= kMaxK, "ance_index_search_exact: need nq >= 0 and 0 < k <= %d", kMaxK);
  if (nq == 0) return ANCE_OK;
  ANCE_REQUIRE(q_dev && D_dev && I_dev, "ance_index_search_exact: null buffer");
  int rc = check_handle_device(ix, "ance_index_search_exact");
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ix->n == 0) {
    // faiss on an empty index: labels -1, scores lowest float
    std::vector<float> d(static_cast<size_t>(nq) * k, -FLT_MAX);
    std::vector<int64_t> i(static_cast<size_t>(nq) * k, -1);
    ANCE_CUDA(cudaMemcpyAsync(D_dev, d.data(), d.size() * 4, cudaMemcpyHostToDevice, st));
    ANCE_CUDA(cudaMemcpyAsync(I_dev, i.data(), i.size() * 8, cudaMemcpyHostToDevice, st));
    ANCE_CUDA(cudaStreamSynchronize(st));
    return ANCE_OK;
  }
  return run_exact(ix, q_dev, nullptr, static_cast<int>(nq), k, D_dev, I_dev, row_offset, st);
}

extern "C" int ance_index_search(ance_index_t ix, const float* q_dev, int64_t nq, int k, float* D_dev,
                                 int64_t* I_dev, int64_t row_offset, void* stream) {
  ANCE_REQUIRE(ix != nullptr, "ance_index_search: null handle");
  ANCE_REQUIRE(nq >= 0 && nq < (1ll << 31), "ance_index_search: nq out of range");
  ANCE_REQUIRE(k > 0, "ance_index_search: k must be positive");
  if (nq == 0) return ANCE_OK;
  ANCE_REQUIRE(q_dev && D_dev && I_dev, "ance_index_search: null buffer");
  int rc = check_handle_device(ix, "ance_index_search");
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ix->last_fetched = 0;
  // choose k' (candidates kept per split).  The certificate needs every row within eps of the k-th score among the
  // candidates; eps is ~0.5 (fp16 operands) / ~3 (bf16) for rows of norm 27.7, i.e. ~0.1 k / ~0.6 k extra rows on the
  // distributions of tools/exp_certify.py.  A query that k' does not cover costs one tier-2 pass, not a wrong answer.
  const bool wide = k > 512;   // the large-k path (kWideCap reservoirs, query blocks)
  int kprime = ix->kprime;
  if (kprime == 0) {
    const int want = (ix->fmt == ANCE_FMT_FP16) ? k + k / 2 - k / 16 : 2 * k + 32;   // fp16: ~1.44 k (k = 200: 288)
    if (!wide)
      kprime = (k <= 240) ? std::min(512, std::max(64, (want + 31) / 32 * 32)) : std::min(992, (2 * k + 31) / 32 * 32);
    else
      kprime = std::min(kWideKPrimeMax, std::max(kWideKPrimeMin, (want + 31) / 32 * 32));
  }
  if (kprime < k || kprime > (wide ? kWideKPrimeMax : 992) || k > kMaxK || ix->n < 4 * static_cast<int64_t>(kprime)) {
    // tiny index or very large k: the exact brute-force path is both correct and cheap enough
    ANCE_REQUIRE(k <= kMaxK, "ance_index_search: k = %d > %d is not supported", k, kMaxK);
    ix->stats = ance_search_stats{};
    ix->stats.nq = nq;
    ix->stats.n_uncertified = nq;
    return ance_index_search_exact(ix, q_dev, nq, k, D_dev, I_dev, row_offset, stream);
  }
  if ((rc = prepare_operands(ix, st))) return rc;
  ance_search_stats acc{};
  if (!wide) {
    rc = search_tiers(ix, q_dev, nq, k, kprime, 992, D_dev, I_dev, row_offset, st, &acc);
    if (rc) return rc;
  } else {
    // Equal blocks of at most kWideQBlock queries (a multiple of the 256-query tile), all tiers per block: the query
    // copies, candidate lists and flagged lists are sized by the block, not by nq.  Tier 2 compacts to kWideKPrimeMax.
    const int64_t n_blocks = (nq + kWideQBlock - 1) / kWideQBlock;
    const int64_t qb = std::min<int64_t>(kWideQBlock, ((nq + n_blocks - 1) / n_blocks + 255) / 256 * 256);
    for (int64_t b0 = 0; b0 < nq; b0 += qb) {
      const int64_t nb = std::min(qb, nq - b0);
      rc = search_tiers(ix, q_dev + b0 * ix->dim, nb, k, kprime, kWideKPrimeMax, D_dev + b0 * k, I_dev + b0 * k,
                        row_offset, st, &acc);
      if (rc) return rc;
    }
  }
  acc.nq = nq;
  acc.kprime = kprime;
  ix->stats = acc;
  ix->last_stream = st;
  return ANCE_OK;
}

extern "C" int ance_index_last_stats(ance_index_t ix, ance_search_stats* out) {
  ANCE_REQUIRE(ix != nullptr && out != nullptr, "ance_index_last_stats: null argument");
  *out = ix->stats;
  return ANCE_OK;
}

extern "C" int ance_index_memory(ance_index_t ix, int64_t* device_bytes, int64_t* host_bytes) {
  ANCE_REQUIRE(ix != nullptr && device_bytes != nullptr && host_bytes != nullptr, "ance_index_memory: null argument");
  const int64_t cap = ix->cap, d = ix->dim;
  int64_t dev = (ix->owns_p32 ? cap * d * 4 : 0) + cap * d * 2 + (ix->ndelta ? cap * 4 : 0);
  dev += 2 * 4 + kMaxPace * 4 + kNumCounters * 4 + d * 4 + d * 8;                       // pstats, pace, counters, mu, colsum
  dev += ix->q_cap * d * 2 + 2 * ix->q_cap * 4;                                          // query operands and norms
  dev += 2 * static_cast<int64_t>(ix->scratch_elems) * 4;                                // coarse reservoirs
  dev += static_cast<int64_t>(ix->cand_ids) * 4 + 2 * static_cast<int64_t>(ix->cand_slots) * 4;   // candidate lists
  dev += 2 * ix->flagged_cap * 4 + static_cast<int64_t>(ix->flagged2_cap) * 4 + static_cast<int64_t>(ix->q16b_elems) * 2;
  dev += static_cast<int64_t>(ix->chunk_keys_elems) * 8;                                 // brute-force keys
  *device_bytes = dev;
  *host_bytes = ix->owns_host ? cap * d * 4 : 0;
  return ANCE_OK;
}

extern "C" int64_t ance_index_last_fetched(ance_index_t ix) { return ix ? ix->last_fetched : -1; }

extern "C" float* ance_index_host_rows(ance_index_t ix) { return (ix && ix->host_rows) ? ix->P32_host : nullptr; }
