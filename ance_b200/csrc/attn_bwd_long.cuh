// attn_bwd_long.cuh — softmax attention backward for dense sequences of 256, 384 or 512 tokens, included by encoder.cu.
//
// The same contract as bwd::attn_bwd_kernel (encoder_bwd.cuh), which holds a whole (sequence, head) in shared memory and
// therefore stops at 128 tokens.  Here the sequence is cut into 64-row blocks and no L x L buffer exists anywhere
// (FlashAttention-2's backward, deterministic, no atomics):
//   dq_kernel   one CTA per (query block, head, sequence).  Pass 1 over the key blocks: S = Q K^T and dP = dO V^T, the
//               online row maximum m and sum l of exp2(s - m), and the running sum of exp2(s - m) dP, which gives
//               D_i = sum_j P_ij dP_ij (the <=128 kernel's rowsum: no read of the 16-bit O, and every row of dS sums to
//               zero up to rounding).  m, 1/l and D go to `stats`.  Pass 2 rebuilds P = exp2(s - m) / l and
//               dS / 8 = P (dP - D) / 8 and accumulates dQ = (dS / 8) K.
//   dkv_kernel  one CTA per (key block, head, sequence), after dq_kernel: for every query block it rebuilds S^T, P^T and
//               dP^T from the stats and accumulates dV = P^T dO and dK = (dS / 8)^T Q in registers.
// Scores are in log2 units with the key bias added, as the forward forms them: s = fmaf(q.k, log2(e) / 8, kbias).
// Every product runs on the tensor cores (mma.sync m16n8k16, fp32 accumulation): S in the forward's 16-bit format; dP, dV,
// dK and dQ on bf16 operands (dO is bf16; P and dS / 8 are rounded to bf16 from fp32; with fp16 storage V, Q and K are
// converted to bf16).  Statistics, D and dS are fp32.  No key block is skipped.
// With cls_only only token 0 of a sequence has an upstream gradient: dq_kernel writes zeros for query blocks > 0, and
// dkv_kernel visits query block 0 only.
// Packed row plans (kSeq: seq_row0 / seq_len): sequence b occupies the rows seq_row0[b] .. + seq_len[b] (the grid still
// spans L / 64 blocks, and blocks that start at or past the length exit).  Rows past the length are read as zeros and never
// written, and keys past it take the dense kernel's padding bias, so a row's arithmetic is that of the dense batch.
// Each warp owns 16 rows of its CTA's 64; its products are 16 x 64 accumulator tiles whose fp32 fragments are re-packed
// in registers as the A operand of the next product (the m16n8k16 C and A fragments share their row / column layout).
#pragma once
#include "act16.cuh"
#include "dropout.cuh"

namespace bwdl {

constexpr int kBlk = 64;        // rows of a query or key block
constexpr int kThreads = 128;   // 4 warps x 16 rows
constexpr int kPitch = 72;      // 16-bit elements per shared row: 144 B, so the 8 row addresses of an ldmatrix hit 8 bank groups

// the stats scratch: [B * heads][3][L] fp32 (m, 1 / l, D)
inline size_t stats_floats(int B, int L, int heads) { return static_cast<size_t>(B) * heads * 3 * L; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const uint16_t* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const uint16_t* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

template <uint32_t FMT>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (FMT == tc05::kFmtBF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments of rows row0 .. row0 + 15, columns 0 .. 63 of a shared tile (4 k-steps of 16)
__device__ __forceinline__ void load_a(uint32_t (&a)[4][4], const uint16_t* s, int row0, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) ldsm_x4(a[kk], s + (row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * kPitch + kk * 16 + (lane >> 4) * 8);
}

// c[16 x 64] += a[16 x 64] x^T, x a shared [64 rows][64] tile (row n of x is column n of the product)
template <uint32_t FMT>
__device__ __forceinline__ void mma_abt(float (&c)[8][4], const uint32_t (&a)[4][4], const uint16_t* x, int lane) {
#pragma unroll
  for (int np = 0; np < 4; ++np)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t r[4];
      ldsm_x4(r, x + (np * 16 + (lane & 7) + (lane >> 4) * 8) * kPitch + kk * 16 + ((lane >> 3) & 1) * 8);
      mma16816<FMT>(c[2 * np], a[kk], r[0], r[1]);
      mma16816<FMT>(c[2 * np + 1], a[kk], r[2], r[3]);
    }
}

// c[16 x 64] += a[16 x 64] x, x a shared [64 (k)][64] bf16 tile
__device__ __forceinline__ void mma_ab(float (&c)[8][4], const uint32_t (&a)[4][4], const uint16_t* x, int lane) {
#pragma unroll
  for (int np = 0; np < 4; ++np)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t r[4];
      ldsm_x4_t(r, x + (kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * kPitch + np * 16 + (lane >> 4) * 8);
      mma16816<tc05::kFmtBF16>(c[2 * np], a[kk], r[0], r[1]);
      mma16816<tc05::kFmtBF16>(c[2 * np + 1], a[kk], r[2], r[3]);
    }
}

// the bf16 A operand (16 x 64) of an fp32 accumulator tile, round to nearest
__device__ __forceinline__ void acc_to_a(uint32_t (&a)[4][4], const float (&c)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    a[kk][0] = act16::Act<tc05::kFmtBF16>::pack2(c[2 * kk][0], c[2 * kk][1]);
    a[kk][1] = act16::Act<tc05::kFmtBF16>::pack2(c[2 * kk][2], c[2 * kk][3]);
    a[kk][2] = act16::Act<tc05::kFmtBF16>::pack2(c[2 * kk + 1][0], c[2 * kk + 1][1]);
    a[kk][3] = act16::Act<tc05::kFmtBF16>::pack2(c[2 * kk + 1][2], c[2 * kk + 1][3]);
  }
}

__device__ __forceinline__ void zero(float (&c)[8][4]) {
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) c[n][e] = 0.f;
}

// 64 rows x 64 16-bit columns from global (row r at g + r * ld) into s; with bf != null also a bf16 copy of fp16 values.
// rows >= n_rows are zero.
template <uint32_t FMT>
__device__ __forceinline__ void load_tile(uint16_t* s, uint16_t* bf, const uint16_t* g, size_t ld, int n_rows) {
  for (int i = threadIdx.x; i < kBlk * 8; i += kThreads) {
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < n_rows) v = __ldg(reinterpret_cast<const uint4*>(g + r * ld + c));
    *reinterpret_cast<uint4*>(s + r * kPitch + c) = v;
    if (FMT == tc05::kFmtF16 && bf) {
      uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = act16::Act<tc05::kFmtF16>::unpack2(w[q]);
        w[q] = act16::Act<tc05::kFmtBF16>::pack2(f.x, f.y);
      }
      *reinterpret_cast<uint4*>(bf + r * kPitch + c) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// the dO tile of query block qb: n_rows rows of dout [*, H] from row tok0 + 64 qb, or with cls_only the sequence's single
// row of dout [B, H]
__device__ __forceinline__ void load_dout(uint16_t* s, const uint16_t* dout, int cls_only, int b, size_t tok0, int n_rows,
                                          int qb, int h, int H) {
  if (cls_only) load_tile<tc05::kFmtBF16>(s, nullptr, dout + static_cast<size_t>(b) * H + h * 64, H, qb == 0 ? 1 : 0);
  else load_tile<tc05::kFmtBF16>(s, nullptr, dout + (tok0 + qb * kBlk) * H + h * 64, H, n_rows);
}

// the key bias of key j (kSeq: the plan's, all zero, inside the sequence, the dense padding bias past its length)
template <bool kSeq>
__device__ __forceinline__ float key_bias(const float* kbias, size_t tok0, int j, int len) {
  if constexpr (kSeq) return j < len ? kbias[tok0 + j] : -10000.0f * 1.4426950408889634f;
  return kbias[tok0 + j];
}

// rows of block x (64 x .. 64 x + 63) inside the sequence
template <bool kSeq>
__device__ __forceinline__ int block_rows(int x, int len) {
  if constexpr (kSeq) return min(kBlk, len - x * kBlk);
  return kBlk;
}

// the max and sum over the 4 lanes of a quad (the lanes holding one accumulator row)
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// kDrop: the forward dropped the probabilities with the mask m of site 1 and scale s (dropout.cuh).  Both kernels then
// use dP = m o (dO V^T) s (so D = sum_j P dP) and dkv_kernel P~ = m o P s for dV, the mask regenerated per element.
// dq_kernel: the masked dP of rows (r, r + 8) of key block kb, in place
template <uint32_t FMT, bool kDrop>
__device__ __forceinline__ void drop_dp_rows(float (&dp)[8][4], const drop::Cfg& dc, uint32_t qi0, uint32_t c2, int kb, int t) {
  if constexpr (kDrop) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int half = 0; half < 2; ++half) {   // key chunk 2 kb + half: n = 4 half .. 4 half + 3
        const uint4 w = drop::philox(dc.k0, dc.k1, 4u * (2 * kb + half) + t, qi0 + 8 * hf, c2, dc.stream);
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = dp[4 * half + m][2 * hf + e];
            x = drop::keep(drop::word(w, m), e, dc.thr) ? x * dc.scale : 0.f;
          }
      }
  }
}

// accumulator element (n, e) of lane (g = lane / 4, t = lane % 4) sits at row g + 8 (e / 2), column 8 n + 2 t + e % 2
template <uint32_t FMT, bool kDrop = false, bool kSeq = false>
__global__ void __launch_bounds__(kThreads) dq_kernel(const uint16_t* __restrict__ qkv, const float* __restrict__ kbias,
                                                      const uint16_t* __restrict__ dout, int cls_only,
                                                      float* __restrict__ dqkv, float* __restrict__ stats, int L,
                                                      int heads, float scale_log2, const drop::Cfg dc,
                                                      const int32_t* __restrict__ seq_row0 = nullptr,
                                                      const int32_t* __restrict__ seq_len = nullptr) {
  constexpr bool kConv = FMT == tc05::kFmtF16;
  __shared__ alignas(16) uint16_t sQ[kBlk * kPitch], sO[kBlk * kPitch], sK[kBlk * kPitch], sV[kBlk * kPitch];
  __shared__ alignas(16) uint16_t sKb_[kConv ? kBlk * kPitch : 8];
  __shared__ float sB[kBlk];
  uint16_t* sKb = kConv ? sKb_ : sK;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z, H = heads * 64;
  const int len = kSeq ? seq_len[b] : L;
  if (kSeq && qb * kBlk >= len) return;   // these rows belong to no part of the sequence
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = static_cast<size_t>(3) * H;
  const size_t tok0 = kSeq ? static_cast<size_t>(seq_row0[b]) : static_cast<size_t>(b) * L;
  const int ra = qb * kBlk + warp * 16 + g;                // this lane's rows in the sequence: ra and ra + 8
  const size_t row_a = tok0 + ra;
  if (cls_only && qb > 0) {   // no upstream gradient in this block: dQ = 0
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
        if (!kSeq || ra + 8 * hf < len) *reinterpret_cast<float2*>(dqkv + (row_a + 8 * hf) * ld + h * 64 + n * 8 + 2 * t) = make_float2(0.f, 0.f);
    return;
  }
  load_tile<FMT>(sQ, nullptr, qkv + (tok0 + qb * kBlk) * ld + h * 64, ld, block_rows<kSeq>(qb, len));
  load_dout(sO, dout, cls_only, b, tok0, block_rows<kSeq>(qb, len), qb, h, H);
  __syncthreads();
  uint32_t aQ[4][4], aO[4][4];
  load_a(aQ, sQ, warp * 16, lane);
  load_a(aO, sO, warp * 16, lane);
  const int nkb = kSeq ? (len + kBlk - 1) / kBlk : L / kBlk;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, dn[2] = {0.f, 0.f};
  float s[8][4], dp[8][4];
  // pass 1: m, l and sum_j exp2(s - m) dP over all keys, rescaled at every new maximum
  for (int kb = 0; kb < nkb; ++kb) {
    __syncthreads();
    const uint16_t* kv = qkv + (tok0 + kb * kBlk) * ld + h * 64;
    load_tile<FMT>(sK, nullptr, kv + H, ld, block_rows<kSeq>(kb, len));
    load_tile<FMT>(sV, kConv ? sV : nullptr, kv + 2 * H, ld, block_rows<kSeq>(kb, len));   // V converted to bf16 in place
    if (threadIdx.x < kBlk) sB[threadIdx.x] = key_bias<kSeq>(kbias, tok0, kb * kBlk + threadIdx.x, len);
    __syncthreads();
    zero(s);
    zero(dp);
    mma_abt<FMT>(s, aQ, sK, lane);
    mma_abt<tc05::kFmtBF16>(dp, aO, sV, lane);
    drop_dp_rows<FMT, kDrop>(dp, dc, qb * kBlk + warp * 16 + g, b * heads + h, kb, t);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        s[n][e] = fmaf(s[n][e], scale_log2, sB[n * 8 + 2 * t + (e & 1)]);
        mx[e >> 1] = fmaxf(mx[e >> 1], s[n][e]);
      }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const float mn = fmaxf(m[hf], quad_max(mx[hf]));
      const float alpha = exp2f(m[hf] - mn);
      float ls = 0.f, ds = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = exp2f(s[n][2 * hf + e] - mn);
          ls += p;
          ds = fmaf(p, dp[n][2 * hf + e], ds);
        }
      l[hf] = fmaf(l[hf], alpha, quad_sum(ls));
      dn[hf] = fmaf(dn[hf], alpha, quad_sum(ds));
      m[hf] = mn;
    }
  }
  float inv[2], D[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    inv[hf] = 1.f / l[hf];
    D[hf] = dn[hf] / l[hf];
    if (t == 0) {
      float* st = stats + (static_cast<size_t>(b) * heads + h) * 3 * L + qb * kBlk + warp * 16 + g + 8 * hf;
      st[0] = m[hf];
      st[L] = inv[hf];
      st[2 * L] = D[hf];
    }
  }
  // pass 2: dQ = (dS / 8) K
  float dq[8][4];
  zero(dq);
  for (int kb = 0; kb < nkb; ++kb) {
    __syncthreads();
    const uint16_t* kv = qkv + (tok0 + kb * kBlk) * ld + h * 64;
    load_tile<FMT>(sK, kConv ? sKb : nullptr, kv + H, ld, block_rows<kSeq>(kb, len));
    load_tile<FMT>(sV, kConv ? sV : nullptr, kv + 2 * H, ld, block_rows<kSeq>(kb, len));
    if (threadIdx.x < kBlk) sB[threadIdx.x] = key_bias<kSeq>(kbias, tok0, kb * kBlk + threadIdx.x, len);
    __syncthreads();
    zero(s);
    zero(dp);
    mma_abt<FMT>(s, aQ, sK, lane);
    mma_abt<tc05::kFmtBF16>(dp, aO, sV, lane);
    drop_dp_rows<FMT, kDrop>(dp, dc, qb * kBlk + warp * 16 + g, b * heads + h, kb, t);
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hf = e >> 1;
        const float p = exp2f(fmaf(s[n][e], scale_log2, sB[n * 8 + 2 * t + (e & 1)]) - m[hf]) * inv[hf];
        s[n][e] = p * (dp[n][e] - D[hf]) * 0.125f;
      }
    uint32_t aS[4][4];
    acc_to_a(aS, s);
    mma_ab(dq, aS, sKb, lane);
  }
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
      if (!kSeq || ra + 8 * hf < len)
        *reinterpret_cast<float2*>(dqkv + (row_a + 8 * hf) * ld + h * 64 + n * 8 + 2 * t) = make_float2(dq[n][2 * hf], dq[n][2 * hf + 1]);
}

template <uint32_t FMT, bool kDrop = false, bool kSeq = false>
__global__ void __launch_bounds__(kThreads) dkv_kernel(const uint16_t* __restrict__ qkv, const float* __restrict__ kbias,
                                                       const uint16_t* __restrict__ dout, int cls_only,
                                                       float* __restrict__ dqkv, const float* __restrict__ stats, int L,
                                                       int heads, float scale_log2, const drop::Cfg dc,
                                                       const int32_t* __restrict__ seq_row0 = nullptr,
                                                       const int32_t* __restrict__ seq_len = nullptr) {
  constexpr bool kConv = FMT == tc05::kFmtF16;
  __shared__ alignas(16) uint16_t sQ[kBlk * kPitch], sO[kBlk * kPitch], sK[kBlk * kPitch], sV[kBlk * kPitch];
  __shared__ alignas(16) uint16_t sQb_[kConv ? kBlk * kPitch : 8];
  __shared__ float sM[kBlk], sI[kBlk], sD[kBlk];
  uint16_t* sQb = kConv ? sQb_ : sQ;
  const int kb = blockIdx.x, h = blockIdx.y, b = blockIdx.z, H = heads * 64;
  const int len = kSeq ? seq_len[b] : L;
  if (kSeq && kb * kBlk >= len) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = static_cast<size_t>(3) * H;
  const size_t tok0 = kSeq ? static_cast<size_t>(seq_row0[b]) : static_cast<size_t>(b) * L;
  const uint16_t* kv = qkv + (tok0 + kb * kBlk) * ld + h * 64;
  load_tile<FMT>(sK, nullptr, kv + H, ld, block_rows<kSeq>(kb, len));
  load_tile<FMT>(sV, kConv ? sV : nullptr, kv + 2 * H, ld, block_rows<kSeq>(kb, len));
  __syncthreads();
  uint32_t aK[4][4], aV[4][4];
  load_a(aK, sK, warp * 16, lane);
  load_a(aV, sV, warp * 16, lane);
  const int ka = kb * kBlk + warp * 16 + g;   // this lane's keys in the sequence: ka and ka + 8
  const float kb_r[2] = {key_bias<kSeq>(kbias, tok0, ka, len), key_bias<kSeq>(kbias, tok0, ka + 8, len)};
  const float* st = stats + (static_cast<size_t>(b) * heads + h) * 3 * L;
  float dk[8][4], dv[8][4], s[8][4], dp[8][4];
  zero(dk);
  zero(dv);
  const int nqb = cls_only ? 1 : kSeq ? (len + kBlk - 1) / kBlk : L / kBlk;
  for (int qb = 0; qb < nqb; ++qb) {
    __syncthreads();
    load_tile<FMT>(sQ, kConv ? sQb : nullptr, qkv + (tok0 + qb * kBlk) * ld + h * 64, ld, block_rows<kSeq>(qb, len));
    load_dout(sO, dout, cls_only, b, tok0, block_rows<kSeq>(qb, len), qb, h, H);
    if (threadIdx.x < kBlk) {
      sM[threadIdx.x] = st[qb * kBlk + threadIdx.x];
      sI[threadIdx.x] = st[L + qb * kBlk + threadIdx.x];
      sD[threadIdx.x] = st[2 * L + qb * kBlk + threadIdx.x];
    }
    __syncthreads();
    zero(s);
    zero(dp);
    mma_abt<FMT>(s, aK, sQ, lane);                // S^T: rows = keys, columns = queries
    mma_abt<tc05::kFmtBF16>(dp, aV, sO, lane);    // dP^T
    if constexpr (kDrop) {
      // this lane's keys jr, jr + 8 (jr = kb 64 + warp 16 + g) share one call per query (same 32-key chunk and key pair
      // index); their words are (jr >> 3) & 3 and the next one
      const int jr = kb * kBlk + warp * 16 + g;
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int eq = 0; eq < 2; ++eq) {
          const uint4 w = drop::philox(dc.k0, dc.k1, 4u * (jr >> 5) + ((jr >> 1) & 3), qb * kBlk + n * 8 + 2 * t + eq,
                                       b * heads + h, dc.stream);
#pragma unroll
          for (int hk = 0; hk < 2; ++hk) {
            const int e = 2 * hk + eq;
            const int i = n * 8 + 2 * t + eq;
            const float p = exp2f(fmaf(s[n][e], scale_log2, kb_r[hk]) - sM[i]) * sI[i];
            const bool kp = drop::keep(drop::word(w, ((jr >> 3) & 3) + hk), jr & 1, dc.thr);
            s[n][e] = kp ? p * dc.scale : 0.f;
            dp[n][e] = p * ((kp ? dp[n][e] * dc.scale : 0.f) - sD[i]) * 0.125f;
          }
        }
    } else {
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = n * 8 + 2 * t + (e & 1);
          const float p = exp2f(fmaf(s[n][e], scale_log2, kb_r[e >> 1]) - sM[i]) * sI[i];
          s[n][e] = p;
          dp[n][e] = p * (dp[n][e] - sD[i]) * 0.125f;
        }
    }
    uint32_t aP[4][4];
    acc_to_a(aP, s);
    mma_ab(dv, aP, sO, lane);
    acc_to_a(aP, dp);
    mma_ab(dk, aP, sQb, lane);
  }
  const size_t row_a = tok0 + ka;
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      if (kSeq && ka + 8 * hf >= len) continue;
      float* o = dqkv + (row_a + 8 * hf) * ld + h * 64 + n * 8 + 2 * t;
      *reinterpret_cast<float2*>(o + H) = make_float2(dk[n][2 * hf], dk[n][2 * hf + 1]);
      *reinterpret_cast<float2*>(o + 2 * H) = make_float2(dv[n][2 * hf], dv[n][2 * hf + 1]);
    }
}

}  // namespace bwdl
