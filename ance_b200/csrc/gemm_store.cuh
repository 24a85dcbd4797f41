// gemm_store.cuh — "store" epilogue of the wgmma GEMM: bias, erf-GELU (two closed forms, see gelu_erf2 / gelu_logistic2), residual add, bf16
// output through shared memory + TMA store (or fp32 output by direct stores).  Covers the encoder's
// linear layers K2/K4/K5/K6/K7 of SURVEY.md §2.3 (HF RobertaSelfAttention / RobertaSelfOutput /
// RobertaIntermediate / RobertaOutput reached from model/models.py:150-151, and embeddingHead,
// models.py:152-153) and the debug GEMM used by the bring-up tests.
//
// bf16 path: each group of 4 epilogue warps (= the 128 rows of the tile) turns 64 accumulator columns
// at a time into a 128 x 64 bf16 slab in SWIZZLE_128B shared memory and one thread hands it to the TMA
// (cp.async.bulk.tensor.2d.global.shared::cta); the stores to HBM are then full 128-byte lines and run
// asynchronously under the next slab's math.  Rows / columns past the tensor edge are clipped by TMA.
#pragma once
#include "act16.cuh"
#include "dropout.cuh"
#include "gemm_core.cuh"

namespace gemm {

__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// fp32 pairs held in one 64-bit value: the GELU forms below are written pairwise; each op is the correctly rounded
// scalar fp32 op on both halves.
__device__ __forceinline__ uint64_t pack2(float a, float b) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& a, float& b) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1), unpack2(b, b0, b1), unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1), unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// HF "gelu" = x * 0.5 * (1 + erf(x / sqrt(2))) = relu(x) - 0.5 |x| erfc(|x| / sqrt(2)), with
//   erfc(z) ~= (1 + a1 z + ... + a6 z^6)^-16        (Abramowitz & Stegun 7.1.28, |error| <= 3e-7)
// and the 1/sqrt(2) folded into the coefficients.  |error| of the GELU <= 7.1e-7 absolute (three orders of magnitude
// below the bf16 rounding of the output; tests/test_encoder_refs_cpu.py checks the bound from these coefficients).  The epilogue of the FFN-up GEMM is bound by
// the SFU (MUFU) rate, so this form uses ONE MUFU (rcp) per element and no exponential; everything else is
// FFMA/FMUL: per PAIR of elements 28 fp32 ops + 2 LOP + 2 MUFU.RCP.
__device__ __forceinline__ void gelu_erf2(float& x0, float& x1) {
  const uint64_t x = pack2(x0, x1);
  const uint64_t ax = x & 0x7FFFFFFF7FFFFFFFull;
  uint64_t p = fma2(pack2(5.38297490e-06f, 5.38297490e-06f), ax, pack2(4.88906371e-05f, 4.88906371e-05f));
  p = fma2(p, ax, pack2(3.80035744e-05f, 3.80035744e-05f));
  p = fma2(p, ax, pack2(3.27762635e-03f, 3.27762635e-03f));
  p = fma2(p, ax, pack2(2.11410057e-02f, 2.11410057e-02f));
  p = fma2(p, ax, pack2(4.98673469e-02f, 4.98673469e-02f));
  p = fma2(p, ax, pack2(1.0f, 1.0f));
  p = mul2(p, p);
  p = mul2(p, p);
  p = mul2(p, p);
  p = mul2(p, p);  // (1 + ...)^16 ; overflows to +inf for |x| > ~25, whose reciprocal is the correct 0
  float p0, p1;
  unpack2(p, p0, p1);
  const uint64_t r = pack2(rcp_approx(p0), rcp_approx(p1));
  const uint64_t relu = fma2(ax, pack2(0.5f, 0.5f), mul2(x, pack2(0.5f, 0.5f)));
  unpack2(fma2(mul2(ax, pack2(-0.5f, -0.5f)), r, relu), x0, x1);
}

// The same function in logistic form:  gelu(x) = x * Phi(x) = x / (1 + exp(-g(x))),  g = logit(Phi) fitted by an odd
// degree-9 polynomial (minimax on the GELU itself over |x| <= 8; the leading coefficient is positive, so g -> +-inf
// and the form saturates correctly for any |x|).  |error| <= 3.7e-6 absolute in fp32 (bf16 rounds the result at 2^-9
// relative).  Per PAIR: 16 fp32 ops + 2 MUFU.EX2 + 2 MUFU.RCP  (gelu_erf2: 28 fp32 ops + 2 LOP + 2 MUFU.RCP).
__device__ __forceinline__ void gelu_logistic2(float& x0, float& x1) {
  const uint64_t x = pack2(x0, x1);
  const uint64_t t = mul2(x, x);
  // -log2(e) * (c0 + c1 t + c2 t^2 + c3 t^3 + c4 t^4)
  uint64_t p = fma2(pack2(-3.290565928e-06f, -3.290565928e-06f), t, pack2(8.930850163e-05f, 8.930850163e-05f));
  p = fma2(p, t, pack2(3.548454260e-04f, 3.548454260e-04f));
  p = fma2(p, t, pack2(-1.052178442e-01f, -1.052178442e-01f));
  p = fma2(p, t, pack2(-2.302048445e+00f, -2.302048445e+00f));
  float g0, g1;
  unpack2(mul2(p, x), g0, g1);
  const uint64_t d = fma2(pack2(ex2_approx(g0), ex2_approx(g1)), pack2(1.0f, 1.0f), pack2(1.0f, 1.0f));   // 1 + exp(-g)
  float d0, d1;
  unpack2(d, d0, d1);
  unpack2(mul2(x, pack2(rcp_approx(d0), rcp_approx(d1))), x0, x1);
}

// FMT: 16-bit format of the OUTPUT and of the residual (act16.cuh); the operand format of the GEMM itself is the
// FMT parameter of gemm::launch.  kDrop: dropout between the bias (and activation) and the residual, in fp32 before the
// one rounding: C = m o (A W^T + bias) / (1 - p) + R, the mask of output row r being that of token drop::row_token(r).
template <int BN, int EPI_WARPS, uint32_t FMT = tc05::kFmtBF16, bool kDrop = false>
struct EpStore {
  using A16 = act16::Act<FMT>;
  static constexpr uint64_t kHintA = tc05::kEvictNormal;
  static constexpr uint64_t kHintB = tc05::kEvictLast;  // weights: keep in L2
  static constexpr int kColGroups = EPI_WARPS / 4;
  static constexpr int kColsPerGroup = BN / kColGroups;
  static constexpr int kSlabBytes = BM * 128;            // 128 rows x 64 bf16
  static constexpr int kSmemBytes = kColGroups * kSlabBytes + 64;  // slabs + one residual mbarrier per column group
  static_assert(EPI_WARPS % 4 == 0 && kColsPerGroup % 64 == 0, "epilogue warp layout");

  struct alignas(64) Params {
    CUtensorMap tmC;         // 16-bit output [M, N], box {64, 128}, SWIZZLE_128B (valid when C != null)
    CUtensorMap tmR;         // 16-bit residual, same geometry (valid when R != null and C != null)
    uint16_t* C;             // [M, ldc] 16-bit (FMT) or null
    float* C32;              // [M, ldc32] fp32 or null (direct stores)
    const float* bias;       // [N] or null
    const uint16_t* R;       // residual [M, ldr] (FMT) or null
    int ldc, ldc32, ldr;
    int act;                 // 0 none, 1 gelu (erfc form, |err| <= 7e-7), 2 gelu (logistic form, |err| <= 3.7e-6)
    drop::Cfg drop;          // kDrop only
  };

  uint32_t rphase;

  __device__ __forceinline__ void begin_work(const Params& p, const WorkShape&, const EpiCtx& cx) {
    if (cx.work_seq == 0 && p.R && p.C && !p.C32) {  // residual tiles arrive by TMA: one mbarrier per column group
      const int cgi = cx.epi_warp >> 2;
      uint64_t* rbar = reinterpret_cast<uint64_t*>(cx.ep_smem + kColGroups * kSlabBytes) + cgi;
      if ((cx.epi_warp & 3) == 0 && cx.lane == 0) {
        tc05::mbar_init(rbar, 1);
        tc05::fence_barrier_init();
      }
      tc05::named_bar_sync(2 + cgi, 128);
      rphase = 0;
    }
  }
  __device__ __forceinline__ void end_work(const Params&, const WorkShape&, const EpiCtx&) {}
  __device__ __forceinline__ void end_kernel(const Params& p, const EpiCtx& cx) {
    if (p.C && (cx.epi_warp & 3) == 0 && cx.lane == 0) tc05::bulk_wait_all();
  }

  // bias + activation + residual on one 32-column chunk held as fp32
  __device__ __forceinline__ void finish_chunk(const Params& p, const WorkShape& ws, float (&f)[32], int row,
                                               bool row_ok, int col0, bool direct_residual) {
    const bool full = (col0 + 32 <= ws.N);
    if (p.bias) {
      if (full) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0) + j);
          f[j * 4] += b.x; f[j * 4 + 1] += b.y; f[j * 4 + 2] += b.z; f[j * 4 + 3] += b.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (col0 + i < ws.N) f[i] += __ldg(p.bias + col0 + i);
      }
    }
    if (p.act == 1) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) gelu_erf2(f[i], f[i + 1]);
    } else if (p.act == 2) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) gelu_logistic2(f[i], f[i + 1]);
    }
    if constexpr (kDrop) {
      if (row_ok) {
        const uint32_t t = drop::row_token(p.drop, row);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint4 w = drop::hidden_bits(p.drop, t, static_cast<uint32_t>(col0 >> 3) + k);
#pragma unroll
          for (int i = 0; i < 8; ++i)
            f[8 * k + i] = drop::keep(drop::word(w, i >> 1), i & 1, p.drop.thr) ? f[8 * k + i] * p.drop.scale : 0.f;
        }
      }
    }
    if (direct_residual && p.R && row_ok) {
      const uint16_t* r = p.R + (size_t)row * p.ldr + col0;
      if (full) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 q = __ldg(reinterpret_cast<const uint4*>(r) + j);
          const uint32_t h[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const float2 x = A16::unpack2(h[t]);
            f[j * 8 + t * 2] += x.x;
            f[j * 8 + t * 2 + 1] += x.y;
          }
        }
      } else {
        for (int i = 0; i < 32; ++i)
          if (col0 + i < ws.N) f[i] += A16::to_float(r[i]);
      }
    }
  }

  __device__ __forceinline__ void tile(const Params& p, const WorkShape& ws, const EpiCtx& cx, uint32_t tacc,
                                       int nb) {
    const int cgi = cx.epi_warp >> 2;
    const int r_in_tile = cx.quad * 32 + cx.lane;
    const int row = cx.row0 + r_in_tile;
    const bool row_ok = row < ws.M;
    uint8_t* slab = cx.ep_smem + cgi * kSlabBytes;
    const bool issuer = (cx.epi_warp & 3) == 0 && cx.lane == 0;
#pragma unroll 1
    for (int s = 0; s < kColsPerGroup; s += 64) {
      const int col_in_tile = cgi * kColsPerGroup + s;
      const int col0 = nb * BN + col_in_tile;
      if (col0 >= ws.N) break;  // uniform across the column group
      const bool tma_res = (p.R != nullptr) && (p.C != nullptr) && (p.C32 == nullptr);
      uint64_t* rbar = reinterpret_cast<uint64_t*>(cx.ep_smem + kColGroups * kSlabBytes) + cgi;
      uint8_t* rowp = slab + r_in_tile * 128;
      if (tma_res && issuer) {
        // residual slab -> the staging buffer (free once the previous TMA store has read it)
        tc05::bulk_wait_read_all();
        tc05::mbar_arrive_expect_tx(rbar, kSlabBytes);
        tc05::tma_load_2d(slab, &p.tmR, rbar, col0, cx.row0, tc05::kEvictFirst);
      }
      // Up to 8 epilogue warps: both 32-column halves of the slab are read from the accumulator tile before the first
      // is consumed.  16 warps (fewer registers each): one half at a time.
      constexpr bool kLean = EPI_WARPS > 8;
      uint32_t va[32], vb[kLean ? 1 : 32];
      tc05::acc_ld_x32(tacc + col_in_tile, va);
      if constexpr (!kLean) tc05::acc_ld_x32(tacc + col_in_tile + 32, vb);
      if (!tma_res && p.C) {
        // the slab is free once the previous TMA store has finished reading it
        if (issuer) tc05::bulk_wait_read_all();
        tc05::named_bar_sync(2 + cgi, 128);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float f[32];
        if constexpr (kLean) {
          if (h == 1) {
            tc05::acc_ld_x32(tacc + col_in_tile + 32, va);
          }
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(va[i]);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(h == 0 ? va[i] : vb[i]);
        }
        finish_chunk(p, ws, f, row, row_ok, col0 + h * 32, !tma_res);
        if (p.C32 && row_ok) {
          float* o = p.C32 + (size_t)row * p.ldc32 + col0 + h * 32;
          if (col0 + h * 32 + 32 <= ws.N) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              reinterpret_cast<float4*>(o)[j] = make_float4(f[j * 4], f[j * 4 + 1], f[j * 4 + 2], f[j * 4 + 3]);
          } else {
            for (int i = 0; i < 32; ++i)
              if (col0 + h * 32 + i < ws.N) o[i] = f[i];
          }
        }
        if (p.C) {
          if (tma_res && h == 0) tc05::mbar_wait(rbar, rphase, 20);
#pragma unroll
          for (int q = 0; q < 4; ++q) {  // 16-byte chunk (h*4 + q) of this row, 128-byte swizzle
            uint4* cp = reinterpret_cast<uint4*>(rowp + (((h * 4 + q) ^ (r_in_tile & 7)) * 16));
            if (tma_res) {
              const uint4 rv = *cp;
              const uint32_t rh[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
              for (int t = 0; t < 4; ++t) {
                const float2 x = A16::unpack2(rh[t]);
                f[q * 8 + t * 2] += x.x;
                f[q * 8 + t * 2 + 1] += x.y;
              }
            }
            uint4 o;
            o.x = A16::pack2(f[q * 8 + 0], f[q * 8 + 1]);
            o.y = A16::pack2(f[q * 8 + 2], f[q * 8 + 3]);
            o.z = A16::pack2(f[q * 8 + 4], f[q * 8 + 5]);
            o.w = A16::pack2(f[q * 8 + 6], f[q * 8 + 7]);
            *cp = o;
          }
        }
      }
      if (p.C) {
        if (tma_res) rphase ^= 1;
        tc05::fence_proxy_async_smem();
        tc05::named_bar_sync(2 + cgi, 128);
        if (issuer) {
          tc05::tma_store_2d(&p.tmC, slab, col0, cx.row0);
          tc05::bulk_commit_group();
        }
      }
    }
  }
};

// host helper: output tensor map for EpStore (bf16 [M, N] with row pitch ldc, box 64 x 128, SW128)
inline bool make_store_tmap(CUtensorMap* tm, void* C, int M, int N, int ldc) {
  return tc05_host::make_tmap_2d_16b(tm, C, M, N, ldc, BM, 64);
}

// Epilogue of tc05_gemm_wide_kernel, run from the MMA warpgroup's registers: C = act(acc + bias) + R, 16-bit output
// (FMT) only, no dropout.  Per element it is EpStore's arithmetic in EpStore's order (acc + bias in fp32, the GELU form,
// + the residual converted to fp32, one rounding), so the two give bit-identical outputs.  The GELU costs the tensor
// cores its whole duration here (nothing overlaps this epilogue), so the encoder's FFN-up keeps EpStore.
//
// A warpgroup's 64 x 256 half of the staging buffer is four SWIZZLE_128B slabs of 64 rows x 64 columns, each the box
// of one TMA load (residual) and one TMA store (output).  Slabs past N and halves past M are neither loaded nor stored.
template <uint32_t FMT = tc05::kFmtBF16>
struct EpStoreWide {
  using A16 = act16::Act<FMT>;
  static constexpr uint64_t kHintA = tc05::kEvictNormal;
  static constexpr uint64_t kHintB = tc05::kEvictLast;  // weights: keep in L2
  static constexpr int kSlabBytes = 64 * 128;
  static constexpr int kSmemBytes = 2 * 4 * kSlabBytes;  // 128 x 256 16-bit

  struct alignas(64) Params {
    CUtensorMap tmC;         // 16-bit output [M, N], box {64, 64}, SWIZZLE_128B
    CUtensorMap tmR;         // 16-bit residual, same box (valid when R != null)
    const float* bias;       // [N] or null
    const uint16_t* R;       // residual or null
    int act;                 // as EpStore's
  };

  __device__ static int slabs(const WorkShape& ws, int row0, int col0) {
    return row0 < ws.M ? min(4, (ws.N - col0 + 63) / 64) : 0;
  }

  // stager: the residual of the half at (row0, col0) -> the half, completing on `bar`; without one, just arrive
  __device__ static void fill(const Params& p, const WorkShape& ws, uint8_t* half, uint64_t* bar, int row0, int col0) {
    const int n = p.R ? slabs(ws, row0, col0) : 0;
    if (n == 0) {
      tc05::mbar_arrive(bar);
      return;
    }
    tc05::mbar_arrive_expect_tx(bar, n * kSlabBytes);
    for (int s = 0; s < n; ++s) tc05::tma_load_2d(half + s * kSlabBytes, &p.tmR, bar, col0 + 64 * s, row0, tc05::kEvictFirst);
  }

  // stager: the outputs in the half -> C; returns once the stores have read the half
  __device__ static void drain(const Params& p, const WorkShape& ws, uint8_t* half, int row0, int col0) {
    const int n = slabs(ws, row0, col0);
    for (int s = 0; s < n; ++s) tc05::tma_store_2d(&p.tmC, half + s * kSlabBytes, col0 + 64 * s, row0);
    tc05::bulk_commit_group();
    tc05::bulk_wait_read_all();
  }

  // columns 8j + c, 8j + c + 1 of rows r and r + 8 (j = 8s + i) are one 32-bit word each in 16-byte chunk i of slab s;
  // row r + 8 has row r's swizzle.  The tensor cores idle while this runs, so each slab first issues all its bias and
  // residual loads, then does the arithmetic without branches.
  template <int ACT>
  __device__ __forceinline__ static void slab(const Params& p, const WorkShape& ws, const float* acc, uint8_t* sl,
                                              int col, int r, int c) {
    uint32_t* w0[8];
    float2 b[8];
    uint32_t x0[8], x1[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      w0[i] = reinterpret_cast<uint32_t*>(sl + r * 128 + ((i ^ (r & 7)) << 4) + 2 * c);
      b[i] = (p.bias && col + 8 * i < ws.N) ? __ldg(reinterpret_cast<const float2*>(p.bias + col + 8 * i))
                                            : make_float2(0.f, 0.f);
      x0[i] = p.R ? *w0[i] : 0u;
      x1[i] = p.R ? *(w0[i] + 8 * 128 / 4) : 0u;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v0 = acc[4 * i], v1 = acc[4 * i + 1], v2 = acc[4 * i + 2], v3 = acc[4 * i + 3];
      if (p.bias) {
        v0 += b[i].x; v1 += b[i].y; v2 += b[i].x; v3 += b[i].y;
      }
      if constexpr (ACT == 1) {
        gelu_erf2(v0, v1);
        gelu_erf2(v2, v3);
      } else if constexpr (ACT == 2) {
        gelu_logistic2(v0, v1);
        gelu_logistic2(v2, v3);
      }
      if (p.R) {
        const float2 y0 = A16::unpack2(x0[i]), y1 = A16::unpack2(x1[i]);
        v0 += y0.x; v1 += y0.y; v2 += y1.x; v3 += y1.y;
      }
      *w0[i] = A16::pack2(v0, v1);
      *(w0[i] + 8 * 128 / 4) = A16::pack2(v2, v3);
    }
  }

  // MMA warpgroup: accumulator fragment of m64n256 (tc05.cuh) -> outputs in the half, residual added in place
  __device__ static void tile(const Params& p, const WorkShape& ws, const float (&acc)[128], uint8_t* half, int col0) {
    const int t = threadIdx.x & 127;
    const int r = 16 * (t >> 5) + ((t & 31) >> 2);
    const int c = 2 * (t & 3);
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int col = col0 + 64 * s + c;
      if (p.act == 1) slab<1>(p, ws, acc + 32 * s, half + s * kSlabBytes, col, r, c);
      else if (p.act == 2) slab<2>(p, ws, acc + 32 * s, half + s * kSlabBytes, col, r, c);
      else slab<0>(p, ws, acc + 32 * s, half + s * kSlabBytes, col, r, c);
    }
  }
};

// host helper: output / residual tensor map for EpStoreWide (16-bit [M, N] with row pitch ld, box 64 x 64, SW128)
inline bool make_store_wide_tmap(CUtensorMap* tm, void* C, int M, int N, int ld) {
  return tc05_host::make_tmap_2d_16b(tm, C, M, N, ld, 64, 64);
}

}  // namespace gemm
