// encoder.cu — BERT/RoBERTa-base dual-encoder forward on sm_90a.
//
// Replaces the library calls behind the reference's
//   model/models.py:149-157  RobertaDot_NLL_LN.query_emb/body_emb  (HF RobertaModel -> CLS -> embeddingHead -> norm)
//   model/models.py:165-199  MultiChunk body_emb (caller reshapes [B,2048] -> [4B,512]; token 0 of each chunk)
//   model/models.py:223-259  BiEncoder / HFBertEncoder (CLS of the last layer)
// Per layer (SURVEY.md §2.3 K1-K7):
//   QKV  = X Wqkv^T + b                       wgmma GEMM (gemm_core.cuh), bias epilogue
//   CTX  = softmax(QK^T/8 + mask) V           attention.cuh
//   T    = CTX Wo^T + b + X ; X1 = LN(T)      GEMM with bias+residual epilogue, then ln_rows_kernel
//   F    = gelu_erf(X1 W1^T + b1)             GEMM with bias+GELU epilogue
//   T    = F W2^T + b2 + X1 ; X = LN(T)       GEMM with bias+residual epilogue, then ln_rows_kernel
// Activations and weights are 16-bit in HBM — fp16 by default, bf16 selectable (ance_encoder_config.operand_fmt, see
// act16.cuh) —; embedding tables, biases, LayerNorm parameters, all accumulation, LayerNorm statistics and softmax are
// fp32.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <vector>

#include "attention.cuh"
#include "common.h"
#include "encoder_bwd.cuh"
#include "gemm_store.cuh"

namespace {

constexpr float kLog2e = 1.4426950408889634f;

// ------------------------------------------------------------------------------------------------
// K1: embeddings gather + LayerNorm, position ids, key-bias
// ------------------------------------------------------------------------------------------------
struct EmbedParams {
  const int32_t* ids;    // [B, L]
  const int32_t* lens;   // [B] or null
  const uint8_t* mask;   // [B, L] or null
  int B, L, H;
  int roberta;           // 1: pos = cumsum(ids != pad) * (ids != pad) + pad ; 0: pos = 0..L-1
  int pad_id, vocab, max_pos;
  const float* word;  // [vocab, H]     fp32: the lookup is a gather, not a tensor-core operand, and 3 KB per token
  const float* pos;   // [max_pos, H]   once per forward is noise next to the 24 LayerNorm passes
  const float* type;  // [type_vocab, H] (row 0)
  const float* gamma;
  const float* beta;
  float eps;
  uint16_t* X;           // [B*L, H] 16-bit (FMT)
  float* kbias;          // [B*L]  (1 - mask) * -10000 * log2e
  int* err_flag;
  const int32_t* seq_row0;  // variable-length packing: first packed row of sequence b (null: row b*L); only the
                            // len[b] real tokens are written, kbias is left alone (all zero)
  int long_pad;             // packing: a sequence longer than 128 also writes its padding tokens up to a multiple of
                            // this many rows (0: none), see pack_chunk
};

template <int NV, uint32_t FMT>  // H = NV * 256
__global__ void __launch_bounds__(256) embed_ln_kernel(const EmbedParams p) {
  using A16 = act16::Act<FMT>;
  __shared__ int s_pos[512];
  __shared__ int s_warp_cnt[8];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t* ids = p.ids + static_cast<size_t>(b) * p.L;
  // position ids (L <= 512): inclusive scan of (id != pad)
  for (int base = 0, carry = 0; base < p.L; base += 256) {
    const int t = base + threadIdx.x;
    const int flag = (t < p.L && ids[t] != p.pad_id) ? 1 : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int pre = carry;
    for (int w2 = 0; w2 < warp; ++w2) pre += s_warp_cnt[w2];
    const int incl = pre + __popc(bal & ((2u << lane) - 1u));
    if (t < p.L) s_pos[t] = p.roberta ? (flag ? incl + p.pad_id : p.pad_id) : t;
    int tot = 0;
    for (int w2 = 0; w2 < 8; ++w2) tot += s_warp_cnt[w2];
    carry += tot;
    __syncthreads();
  }
  const int len = p.lens ? p.lens[b] : 0;
  const bool varlen = p.seq_row0 != nullptr;
  const size_t row0 = varlen ? static_cast<size_t>(p.seq_row0[b]) : static_cast<size_t>(b) * p.L;
  const int t_end = !varlen ? p.L : (p.long_pad && len > 128) ? min((len + p.long_pad - 1) / p.long_pad * p.long_pad, p.L) : min(len, p.L);
  for (int t = warp; t < t_end; t += 8) {
    const size_t tok = row0 + t;
    int id = ids[t];
    int ps = s_pos[t];
    if (id < 0 || id >= p.vocab || ps >= p.max_pos) {
      if (lane == 0) atomicOr(p.err_flag, 1);
      id = min(max(id, 0), p.vocab - 1);
      ps = min(ps, p.max_pos - 1);
    }
    const float4* wr = reinterpret_cast<const float4*>(p.word + static_cast<size_t>(id) * p.H);
    const float4* pr = reinterpret_cast<const float4*>(p.pos + static_cast<size_t>(ps) * p.H);
    const float4* tr = reinterpret_cast<const float4*>(p.type);
    float x[NV * 8];
    float sum = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {   // the same (word + pos) + type association as the reference's embeddings sum
        const int c4 = (v * 32 + lane) * 2 + hf;
        const float4 a = __ldg(wr + c4), c = __ldg(pr + c4), d = __ldg(tr + c4);
        x[v * 8 + hf * 4 + 0] = (a.x + c.x) + d.x;
        x[v * 8 + hf * 4 + 1] = (a.y + c.y) + d.y;
        x[v * 8 + hf * 4 + 2] = (a.z + c.z) + d.z;
        x[v * 8 + hf * 4 + 3] = (a.w + c.w) + d.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) sum += x[v * 8 + i];
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    const float mean = sum / p.H;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < NV * 8; ++i) {
      const float dlt = x[i] - mean;
      var = fmaf(dlt, dlt, var);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
    const float rstd = rsqrtf(var / p.H + p.eps);
    uint4* out = reinterpret_cast<uint4*>(p.X + tok * p.H);
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * 32 + lane) * 8;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(p.gamma + col)), g1 = __ldg(reinterpret_cast<const float4*>(p.gamma + col + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.beta + col)), b1 = __ldg(reinterpret_cast<const float4*>(p.beta + col + 4));
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint32_t h2[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        h2[q] = A16::pack2((x[v * 8 + q * 2] - mean) * rstd * g[q * 2] + bb[q * 2],
                           (x[v * 8 + q * 2 + 1] - mean) * rstd * g[q * 2 + 1] + bb[q * 2 + 1]);
      out[v * 32 + lane] = make_uint4(h2[0], h2[1], h2[2], h2[3]);
    }
    if (lane == 0 && !varlen) {
      const bool keep = p.mask ? (p.mask[tok] != 0) : (t < len);
      p.kbias[tok] = keep ? 0.f : -10000.0f * kLog2e;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over rows: 16-bit (FMT) or fp32 in, 16-bit and/or fp32 out; row r read at in + r * in_ld
// ------------------------------------------------------------------------------------------------
template <int NV, bool kInF32, uint32_t FMT>
__global__ void __launch_bounds__(256) ln_rows_kernel(const void* __restrict__ in, size_t in_ld, int n_rows, int H,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      float eps, uint16_t* __restrict__ out16,
                                                      float* __restrict__ out32) {
  using A16 = act16::Act<FMT>;
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  float x[NV * 8];
  float sum = 0.f;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * 32 + lane) * 8;
    if (kInF32) {
      const float* r = reinterpret_cast<const float*>(in) + static_cast<size_t>(row) * in_ld + col;
      const float4 a = __ldg(reinterpret_cast<const float4*>(r)), b = __ldg(reinterpret_cast<const float4*>(r + 4));
      x[v * 8 + 0] = a.x; x[v * 8 + 1] = a.y; x[v * 8 + 2] = a.z; x[v * 8 + 3] = a.w;
      x[v * 8 + 4] = b.x; x[v * 8 + 5] = b.y; x[v * 8 + 6] = b.z; x[v * 8 + 7] = b.w;
    } else {
      const uint16_t* r = reinterpret_cast<const uint16_t*>(in) + static_cast<size_t>(row) * in_ld + col;
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(r));
      const uint32_t ah[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = A16::unpack2(ah[q]);
        x[v * 8 + q * 2] = f.x;
        x[v * 8 + q * 2 + 1] = f.y;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) sum += x[v * 8 + i];
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  const float mean = sum / H;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < NV * 8; ++i) {
    const float d = x[i] - mean;
    var = fmaf(d, d, var);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
  const float rstd = rsqrtf(var / H + eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * 32 + lane) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + col)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + col)), b1 = __ldg(reinterpret_cast<const float4*>(beta + col + 4));
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float y[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = (x[v * 8 + i] - mean) * rstd * g[i] + bb[i];
    if (out16) {
      *reinterpret_cast<uint4*>(out16 + static_cast<size_t>(row) * H + col) =
          make_uint4(A16::pack2(y[0], y[1]), A16::pack2(y[2], y[3]), A16::pack2(y[4], y[5]), A16::pack2(y[6], y[7]));
    }
    if (out32) {
      float* o = out32 + static_cast<size_t>(row) * H + col;
      *reinterpret_cast<float4*>(o) = make_float4(y[0], y[1], y[2], y[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(y[4], y[5], y[6], y[7]);
    }
  }
}

// 16-bit -> 16-bit LayerNorm, kB rows per warp written as independent instruction streams (their shuffle / FMA chains
// overlap and gamma / beta are fetched once); the arithmetic of a row is that of ln_rows_kernel, bit for bit.
template <int NV, int kB, uint32_t FMT>
__global__ void __launch_bounds__(256) ln_rows_multi_kernel(const uint16_t* __restrict__ in, size_t in_ld, int n_rows, int H,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float eps, uint16_t* __restrict__ out16) {
  using A16 = act16::Act<FMT>;
  const int lane = threadIdx.x & 31;
  const int row0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * kB;
  if (row0 >= n_rows) return;
  float x[kB][NV * 8], sum[kB], var[kB], mean[kB], rstd[kB];
#pragma unroll
  for (int b = 0; b < kB; ++b) {
    const int row = min(row0 + b, n_rows - 1);
    const uint4* src = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * in_ld);
    uint4 raw[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) raw[v] = __ldg(src + v * 32 + lane);
    sum[b] = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const uint32_t ah[4] = {raw[v].x, raw[v].y, raw[v].z, raw[v].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = A16::unpack2(ah[q]);
        x[b][v * 8 + q * 2] = f.x;
        x[b][v * 8 + q * 2 + 1] = f.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) sum[b] += x[b][v * 8 + i];
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int b = 0; b < kB; ++b) sum[b] += __shfl_xor_sync(0xffffffffu, sum[b], s);
  }
#pragma unroll
  for (int b = 0; b < kB; ++b) {
    mean[b] = sum[b] / H;
    var[b] = 0.f;
#pragma unroll
    for (int i = 0; i < NV * 8; ++i) {
      const float d = x[b][i] - mean[b];
      var[b] = fmaf(d, d, var[b]);
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int b = 0; b < kB; ++b) var[b] += __shfl_xor_sync(0xffffffffu, var[b], s);
  }
#pragma unroll
  for (int b = 0; b < kB; ++b) rstd[b] = rsqrtf(var[b] / H + eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * 32 + lane) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + col)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + col)), b1 = __ldg(reinterpret_cast<const float4*>(beta + col + 4));
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int b = 0; b < kB; ++b) {
      float y[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = (x[b][v * 8 + i] - mean[b]) * rstd[b] * g[i] + bb[i];
      const uint4 u = make_uint4(A16::pack2(y[0], y[1]), A16::pack2(y[2], y[3]), A16::pack2(y[4], y[5]), A16::pack2(y[6], y[7]));
      if (row0 + b < n_rows) *reinterpret_cast<uint4*>(out16 + static_cast<size_t>(row0 + b) * H + col) = u;
    }
  }
}

// rows r*stride of a 16-bit matrix -> fp32 [n, H]   (DPR: CLS of the last layer, models.py:239)
template <uint32_t FMT>
__global__ void gather_rows_f32_kernel(const uint16_t* __restrict__ X, size_t row_stride, int n, int H,
                                       float* __restrict__ out) {
  const int r = blockIdx.x;
  for (int c = threadIdx.x; c < H; c += blockDim.x)
    out[static_cast<size_t>(r) * H + c] = act16::Act<FMT>::to_float(X[static_cast<size_t>(r) * row_stride + c]);
}

// Same arithmetic again (bit-identical), holding the rows PACKED: kB x NV uint4 registers instead of kB x NV x 8 floats; the
// three passes (sum, variance, normalise) unpack on the fly.  ~56 instead of 83 registers per thread -> 4 instead of 3
// resident blocks per SM (the float form is latency-bound, well below the HBM roof).
template <int NV, int kB, uint32_t FMT>
__global__ void __launch_bounds__(256, 4) ln_rows_packed_kernel(const uint16_t* __restrict__ in, size_t in_ld, int n_rows, int H,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                float eps, uint16_t* __restrict__ out16) {
  using A16 = act16::Act<FMT>;
  const int lane = threadIdx.x & 31;
  const int row0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * kB;
  if (row0 >= n_rows) return;
  uint4 raw[kB][NV];
  float sum[kB], var[kB], mean[kB], rstd[kB];
#pragma unroll
  for (int b = 0; b < kB; ++b) {
    const int row = min(row0 + b, n_rows - 1);
    const uint4* src = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * in_ld);
#pragma unroll
    for (int v = 0; v < NV; ++v) raw[b][v] = __ldg(src + v * 32 + lane);
  }
#pragma unroll
  for (int b = 0; b < kB; ++b) {
    sum[b] = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const uint32_t w[4] = {raw[b][v].x, raw[b][v].y, raw[b][v].z, raw[b][v].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {   // same order as ln_rows_multi_kernel: x[8v + 2q], x[8v + 2q + 1]
        const float2 f = A16::unpack2(w[q]);
        sum[b] += f.x;
        sum[b] += f.y;
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int b = 0; b < kB; ++b) sum[b] += __shfl_xor_sync(0xffffffffu, sum[b], s);
  }
#pragma unroll
  for (int b = 0; b < kB; ++b) {
    mean[b] = sum[b] / H;
    var[b] = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const uint32_t w[4] = {raw[b][v].x, raw[b][v].y, raw[b][v].z, raw[b][v].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = A16::unpack2(w[q]);
        const float d0 = f.x - mean[b], d1 = f.y - mean[b];
        var[b] = fmaf(d0, d0, var[b]);
        var[b] = fmaf(d1, d1, var[b]);
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
    for (int b = 0; b < kB; ++b) var[b] += __shfl_xor_sync(0xffffffffu, var[b], s);
  }
#pragma unroll
  for (int b = 0; b < kB; ++b) rstd[b] = rsqrtf(var[b] / H + eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * 32 + lane) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + col)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + col)), b1 = __ldg(reinterpret_cast<const float4*>(beta + col + 4));
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int b = 0; b < kB; ++b) {
      const uint32_t w[4] = {raw[b][v].x, raw[b][v].y, raw[b][v].z, raw[b][v].w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = A16::unpack2(w[q]);
        o[q] = A16::pack2((f.x - mean[b]) * rstd[b] * g[q * 2] + bb[q * 2], (f.y - mean[b]) * rstd[b] * g[q * 2 + 1] + bb[q * 2 + 1]);
      }
      if (row0 + b < n_rows) *reinterpret_cast<uint4*>(out16 + static_cast<size_t>(row0 + b) * H + col) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// rows idx[r] of a 16-bit matrix [*, H] -> compact [n, H]  (variable-length packing: the CLS rows sit at arbitrary rows)
__global__ void gather_rows16_by_index_kernel(const uint16_t* __restrict__ src, const int32_t* __restrict__ idx, int n, int H,
                                              uint16_t* __restrict__ dst) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(idx[r]) * H);
  uint4* o = reinterpret_cast<uint4*>(dst + static_cast<size_t>(r) * H);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) o[i] = __ldg(s + i);
}

template <uint32_t FMT>
__global__ void act16_to_f32_kernel(const uint16_t* __restrict__ in, float* __restrict__ out, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = act16::Act<FMT>::to_float(in[i]);
}

// any non-finite value in the final embeddings (fp16 overflow somewhere upstream, or NaN weights) -> err_flag bit 1
__global__ void check_finite_kernel(const float* __restrict__ x, size_t n, int* __restrict__ err_flag) {
  bool bad = false;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    bad |= !(fabsf(x[i]) <= 3.0e38f);
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(err_flag, 2);
}

}  // namespace

// ================================================================================================
// handle
// ================================================================================================
struct LayerDev {
  uint16_t *wqkv, *wo, *w1, *w2;         // [3H,H] [H,H] [F,H] [H,F]  16-bit (fmt)
  float *bqkv, *bo, *b1, *b2, *ln1g, *ln1b, *ln2g, *ln2b;
};

struct ance_encoder {
  ance_encoder_config cfg{};
  int max_tokens = 0;
  uint32_t fmt = tc05::kFmtF16;          // 16-bit storage format of activations and weights
  int device = 0;
  float *word = nullptr, *pos = nullptr, *type = nullptr;
  float *eg = nullptr, *eb = nullptr;
  std::vector<LayerDev> layers;
  uint16_t* head_w = nullptr;
  float *head_b = nullptr, *head_g = nullptr, *head_bt = nullptr;
  // activations
  uint16_t *X = nullptr, *QKV = nullptr, *CTX = nullptr, *T = nullptr, *X1 = nullptr, *FF = nullptr;
  float* kbias = nullptr;
  uint16_t *cls_ctx = nullptr, *cls_x = nullptr;   // [max_seqs, H]: CLS rows gathered for the pruned last layer (varlen)
  int32_t* seq_row0 = nullptr;                     // [max_seqs] varlen plan: first packed row of each sequence
  int32_t *row_lo = nullptr, *row_hi = nullptr;    // [max_tokens] varlen plan: own-sequence key range of each packed row
  int2* tile_kv = nullptr;                         // [max_tokens / 128] varlen plan: key blocks of each tile
  float* head_tmp = nullptr;  // [max_seqs, H] fp32
  int* err_flag = nullptr;
  uint16_t* dbg = nullptr;       // [(n_layer+1), max_tokens, H] when debugging
  int dbg_tokens = 0;
  int prune_last_layer = 1;  // last layer: only the CLS rows go through out-proj / FFN (identical result)
  int varlen_align = 1;      // ance_encoder_forward_varlen / _packed: 1 = densest, 16 = exact packing, see pack_chunk
  std::vector<void*> allocs;
  // training (ance_encoder_forward_train / _backward)
  std::map<const void*, int2> train_shapes;   // workspace -> (B, L) of a forward_train whose backward has not run yet
  struct LayerT { uint16_t *wqkv, *wo, *w1, *w2; };   // bf16 W^T: [H,3H] [H,H] [H,F] [F,H]
  std::vector<LayerT> wt;                     // empty until the first backward
  uint16_t* head_wt = nullptr;
  bool wt_stale = true;                       // the W^T copies no longer match the weights
  void* bwd_scratch = nullptr;                // backward scratch (ance_encoder_destroy frees it)
  std::vector<bwd::RefreshPiece> refresh_table;   // ance_encoder_update_weights: the last table uploaded
  bwd::RefreshPiece* refresh_dev = nullptr;       // its device copy (ance_encoder_destroy frees it)
  size_t refresh_cap = 0;
  size_t bwd_scratch_bytes = 0;
};

namespace {

// ANCE_ERR_CUDA unless the current device is an sm_90 GPU (there is no CPU fallback)
int require_sm90(int* dev_out) {
  int dev = 0, major = 0, minor = 0;
  ANCE_CUDA(cudaGetDevice(&dev));
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    ance::set_error("device %d has compute capability %d.%d; libance_b200 is built for sm_90a only (no CPU fallback)", dev, major, minor);
    return ANCE_ERR_CUDA;
  }
  if (dev_out) *dev_out = dev;
  return ANCE_OK;
}

template <class T>
T* dev_alloc(ance_encoder* e, size_t n) {
  void* p = nullptr;
  if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) return nullptr;
  e->allocs.push_back(p);
  return reinterpret_cast<T*>(p);
}

float* upload_f32(ance_encoder* e, const float* h, size_t n) {
  float* d = dev_alloc<float>(e, n);
  if (d) cudaMemcpy(d, h, n * 4, cudaMemcpyHostToDevice);
  return d;
}

uint16_t* upload_16(ance_encoder* e, const float* h, size_t n) {
  std::vector<uint16_t> tmp(n);
  if (e->fmt == tc05::kFmtBF16) for (size_t i = 0; i < n; ++i) tmp[i] = act16::Act<tc05::kFmtBF16>::from_float_host(h[i]);
  else for (size_t i = 0; i < n; ++i) tmp[i] = act16::Act<tc05::kFmtF16>::from_float_host(h[i]);
  uint16_t* d = dev_alloc<uint16_t>(e, n);
  if (d) cudaMemcpy(d, tmp.data(), n * 2, cudaMemcpyHostToDevice);
  return d;
}

// GELU form of the FFN-up epilogue: 2 = logistic form (|err| <= 3.7e-6), 1 = erfc form (|err| <= 7.1e-7)
int gelu_form() {
  static const int form = getenv("ANCE_B200_GELU") ? atoi(getenv("ANCE_B200_GELU")) : 2;
  return form;
}

// one GEMM of the forward: C[M,N] = act(A[M,K] W[N,K]^T + bias) (+ R); act is the epilogue's code: 0 none, 1 / 2 GELU
// (see gelu_form).  128 x 128 tile per CTA (the wgmma warpgroup holds the whole tile in registers: 128 fp32 accumulators
// per thread), 4 operand stages, 4 epilogue warps reading the shared accumulator tile while the next tile is computed.
template <uint32_t FMT>
int linear(const uint16_t* A, size_t lda, int M, const uint16_t* W, int N, int K, const float* bias,
           const uint16_t* R, int act, uint16_t* C, float* C32, cudaStream_t st, int cls = ance::kClsGemm,
           size_t ldr = 0) {
  constexpr int BN = 128, CG = 1, EW = 4, STAGES = 4;
  using Ep = gemm::EpStore<BN, EW, FMT>;
  CUtensorMap tmA, tmB;
  if (!tc05_host::make_tmap_2d_16b(&tmA, A, M, K, lda, gemm::BM) || !tc05_host::make_tmap_2d_16b(&tmB, W, N, K, K, BN / CG)) {
    ance::set_error("encoder: cuTensorMapEncodeTiled failed (M=%d N=%d K=%d)", M, N, K);
    return ANCE_ERR_CUDA;
  }
  gemm::WorkShape ws = gemm::make_shape(M, N, K, BN, CG, 0);
  typename Ep::Params p;
  memset(&p, 0, sizeof(p));
  if (C && !gemm::make_store_tmap(&p.tmC, C, M, N, N)) {
    ance::set_error("encoder: cuTensorMapEncodeTiled failed for the output (M=%d N=%d)", M, N);
    return ANCE_ERR_CUDA;
  }
  if (ldr == 0) ldr = N;
  if (C && R && !gemm::make_store_tmap(&p.tmR, const_cast<uint16_t*>(R), M, N, static_cast<int>(ldr))) {
    ance::set_error("encoder: cuTensorMapEncodeTiled failed for the residual (M=%d N=%d)", M, N);
    return ANCE_ERR_CUDA;
  }
  p.C = C;
  p.C32 = C32;
  p.bias = bias;
  p.R = R;
  p.ldc = N;
  p.ldc32 = N;
  p.ldr = static_cast<int>(ldr);
  p.act = act;
  {
    ance::ProfScope ps(cls, st);
    ANCE_CUDA((gemm::launch<Ep, BN, STAGES, CG, EW, FMT>(tmA, tmB, ws, p, 0, st)));
  }
  ance::count_launch(1);
  return ANCE_OK;
}

int g_ln_rows_per_warp = 2;   // ance_encoder_set_param("ln_rows_per_warp")

template <uint32_t FMT>
int layer_norm(const void* in, bool in_f32, size_t in_ld, int rows, int H, const float* g, const float* b, float eps,
               uint16_t* out16, float* out32, cudaStream_t st) {
  const int blocks = (rows + 7) / 8;
  const int nv = H / 256;
  ance::ProfScope ps(ance::kClsNorm, st);
  if (!in_f32 && out16 && !out32 && nv == 3 && g_ln_rows_per_warp > 1 && rows >= 4096) {
    const uint16_t* src = reinterpret_cast<const uint16_t*>(in);
    if (g_ln_rows_per_warp == 2) ln_rows_multi_kernel<3, 2, FMT><<<(rows + 15) / 16, 256, 0, st>>>(src, in_ld, rows, H, g, b, eps, out16);
    else if (g_ln_rows_per_warp == 3) ln_rows_packed_kernel<3, 2, FMT><<<(rows + 15) / 16, 256, 0, st>>>(src, in_ld, rows, H, g, b, eps, out16);   // 2 rows, packed registers
    else ln_rows_multi_kernel<3, 4, FMT><<<(rows + 31) / 32, 256, 0, st>>>(src, in_ld, rows, H, g, b, eps, out16);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
    return ANCE_OK;
  }
#define LN_CASE(NV_)                                                                                            \
  if (in_f32) ln_rows_kernel<NV_, true, FMT><<<blocks, 256, 0, st>>>(in, in_ld, rows, H, g, b, eps, out16, out32); \
  else ln_rows_kernel<NV_, false, FMT><<<blocks, 256, 0, st>>>(in, in_ld, rows, H, g, b, eps, out16, out32)
  if (nv == 3) { LN_CASE(3); }
  else if (nv == 4) { LN_CASE(4); }
  else if (nv == 1) { LN_CASE(1); }
  else if (nv == 2) { LN_CASE(2); }
  else { ance::set_error("encoder: hidden size %d unsupported", H); return ANCE_ERR_UNSUPPORTED; }
#undef LN_CASE
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

template <uint32_t FMT>
int set_attention_attrs() {
  // per device, not per process: a second GPU used from the same process needs its own opt-in
  ANCE_CUDA(cudaFuncSetAttribute(attn::attention_kernel<false, false, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::Smem::kDynamic));
  ANCE_CUDA(cudaFuncSetAttribute(attn::attention_kernel<false, true, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::Smem::kDynamic));
  ANCE_CUDA(cudaFuncSetAttribute(attn::attention_kernel<true, true, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::Smem::kDynamic));
  ANCE_CUDA(cudaFuncSetAttribute(attn::attention_kernel<true, false, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::Smem::kDynamic));
  return ANCE_OK;
}

// The attention of one layer: ctx [n_tokens, 64 heads] = softmax(Q K^T / 8 + kbias) V over qkv [n_tokens, 3 * 64 heads].
// Dense (row_lo null): sequences of L tokens back to back.  Variable-length packing (row_lo / row_hi, and tile_kv when
// L > 128, see PackPlan): n_tokens = 128 * tiles.  Built once per forward, launched once per layer.
struct AttentionLaunch {
  CUtensorMap tmQKV, tmCTX;
  attn::Params ap;
  int grid;
  bool packed, single;   // the attention_kernel<kPacked, kSingle> instantiation
};

int make_attention(AttentionLaunch& a, const uint16_t* qkv, uint16_t* ctx, int n_tokens, int L, int heads,
                   const float* kbias, const int32_t* row_lo, const int32_t* row_hi, const int2* tile_kv) {
  const int H = heads * attn::kDh;
  if (!tc05_host::make_tmap_2d_16b(&a.tmQKV, qkv, n_tokens, 3 * H, 3 * H, attn::kTile)) {
    ance::set_error("encoder: cuTensorMapEncodeTiled failed for QKV");
    return ANCE_ERR_CUDA;
  }
  if (!tc05_host::make_tmap_2d_16b(&a.tmCTX, ctx, n_tokens, H, H, attn::kTile)) {
    ance::set_error("encoder: cuTensorMapEncodeTiled failed for the attention output");
    return ANCE_ERR_CUDA;
  }
  const bool varlen = row_lo != nullptr;
  const bool varlen_long = varlen && L > attn::kTile;   // sequences may span several tiles: multi-block attention items
  attn::Params& ap = a.ap;
  ap.n_tokens = n_tokens; ap.L = (varlen && !varlen_long) ? 64 : L; ap.heads = heads; ap.hidden = H;   // varlen: any L < 128 selects the packed kernel
  ap.kbias = kbias;
  ap.scale_log2 = kLog2e / 8.0f;
  ap.row_lo = varlen ? row_lo : nullptr;
  ap.row_hi = varlen ? row_hi : nullptr;
  ap.tile_kv = varlen ? tile_kv : nullptr;
  const int attn_work = ((n_tokens + 127) / 128) * heads;
  a.grid = std::min(attn_work, gemm::sm_count());
  a.packed = varlen || L < attn::kTile;
  a.single = !varlen_long && L <= attn::kTile;
  return ANCE_OK;
}

template <uint32_t FMT>
int run_attention(const AttentionLaunch& a, cudaStream_t st) {
  ance::prof_begin(ance::kClsAttn, st);
  if (a.packed && !a.single) attn::attention_kernel<true, false, FMT><<<a.grid, attn::kThreads, attn::Smem::kDynamic, st>>>(a.tmQKV, a.tmCTX, a.ap);
  else if (a.packed) attn::attention_kernel<true, true, FMT><<<a.grid, attn::kThreads, attn::Smem::kDynamic, st>>>(a.tmQKV, a.tmCTX, a.ap);
  else if (a.single) attn::attention_kernel<false, true, FMT><<<a.grid, attn::kThreads, attn::Smem::kDynamic, st>>>(a.tmQKV, a.tmCTX, a.ap);
  else attn::attention_kernel<false, false, FMT><<<a.grid, attn::kThreads, attn::Smem::kDynamic, st>>>(a.tmQKV, a.tmCTX, a.ap);
  ance::prof_end(ance::kClsAttn, st);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

// What the training forward keeps for the backward, in the caller's workspace (M = B * L tokens, byte offsets):
//   ids [M] int32, kbias [M] fp32, then per layer the layer input X, QKV, CTX (M rows) and the LayerNorm inputs T1 / T2,
//   the LayerNorm-1 output X1, the FFN-up pre-activation U and GELU output FF (M rows reserved, B used in the pruned last
//   layer), then the last layer's CLS outputs [B, H] and the head LayerNorm's fp32 input [B, H].  Activations are 16-bit
//   (operand_fmt).  LayerNorm statistics and softmax statistics are not stored: the backward recomputes them.
struct TrainLayout {
  size_t ids, kbias, layers, per_layer, x_in, qkv, ctx, t1, x1, u, ff, t2, x_final, head_in, total;
};

TrainLayout train_layout(const ance_encoder_config& c, int B, int L) {
  const size_t M = static_cast<size_t>(B) * L, H = c.hidden, F = c.ffn;
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  TrainLayout t;
  size_t o = 0;
  t.ids = o; o += up(M * 4);
  t.kbias = o; o += up(M * 4);
  t.layers = o;
  size_t p = 0;
  t.x_in = p; p += up(M * H * 2);
  t.qkv = p; p += up(M * 3 * H * 2);
  t.ctx = p; p += up(M * H * 2);
  t.t1 = p; p += up(M * H * 2);
  t.x1 = p; p += up(M * H * 2);
  t.u = p; p += up(M * F * 2);
  t.ff = p; p += up(M * F * 2);
  t.t2 = p; p += up(M * H * 2);
  t.per_layer = p;
  o += p * c.n_layer;
  t.x_final = o; o += up(static_cast<size_t>(B) * H * 2);
  t.head_in = o; o += up(static_cast<size_t>(B) * H * 4);
  t.total = o;
  return t;
}

struct TrainSave {
  uint8_t* ws;
  TrainLayout lo;
  int n_layer;
  uint16_t* at(int l, size_t off) const { return reinterpret_cast<uint16_t*>(ws + lo.layers + l * lo.per_layer + off); }
  uint16_t* x(int l) const { return l == n_layer ? reinterpret_cast<uint16_t*>(ws + lo.x_final) : at(l, lo.x_in); }
  int32_t* ids() const { return reinterpret_cast<int32_t*>(ws + lo.ids); }
  float* kbias() const { return reinterpret_cast<float*>(ws + lo.kbias); }
  float* head_in() const { return reinterpret_cast<float*>(ws + lo.head_in); }
};

// n_tiles > 0: variable-length packing — the plan (e->seq_row0 / row_lo / row_hi / tile_kv) is already on the device, the
// token matrix has n_tiles * 128 rows and the CLS rows are gathered by index.  With L > 128 sequences may span tiles.
// ts != null (dense, L <= 128): the training forward — the same launches on the same inputs, with every activation the
// backward needs written to its own slot of the workspace instead of the reused buffers of the handle (plus the FFN-up
// GEMM once more without GELU for the pre-activation), and the last layer always pruned to the CLS rows.
template <uint32_t FMT>
int forward_impl(ance_encoder* e, const int32_t* ids_dev, const int32_t* lens_dev, const uint8_t* mask_dev, int B, int L,
                 float* out_dev, cudaStream_t st, int n_tiles = 0, const TrainSave* ts = nullptr) {
  const ance_encoder_config& c = e->cfg;
  const bool varlen = n_tiles > 0;
  const bool varlen_long = varlen && L > attn::kTile;   // sequences may span several tiles: multi-block attention items
  const int M = varlen ? n_tiles * attn::kTile : B * L, H = c.hidden, F = c.ffn;
  int rc;
  if (varlen) {   // rows behind the last sequence of a tile: zeros (finite through every layer), no key bias anywhere
    ANCE_CUDA(cudaMemsetAsync(e->X, 0, static_cast<size_t>(M) * H * 2, st));
    ANCE_CUDA(cudaMemsetAsync(e->kbias, 0, static_cast<size_t>(M) * 4, st));
  }
  // K1
  EmbedParams ep;
  if (ts) ANCE_CUDA(cudaMemcpyAsync(ts->ids(), ids_dev, static_cast<size_t>(M) * 4, cudaMemcpyDeviceToDevice, st));
  ep.ids = ids_dev; ep.lens = lens_dev; ep.mask = mask_dev;
  ep.B = B; ep.L = L; ep.H = H;
  ep.roberta = (c.arch == ANCE_ARCH_ROBERTA);
  ep.pad_id = c.pad_id; ep.vocab = c.vocab; ep.max_pos = c.max_pos;
  ep.word = e->word; ep.pos = e->pos; ep.type = e->type;
  ep.gamma = e->eg; ep.beta = e->eb; ep.eps = c.ln_eps;
  ep.X = ts ? ts->x(0) : e->X; ep.kbias = ts ? ts->kbias() : e->kbias; ep.err_flag = e->err_flag;
  ep.seq_row0 = varlen ? e->seq_row0 : nullptr;
  ep.long_pad = (varlen_long && e->varlen_align == 16) ? 32 : 0;
  ance::prof_begin(ance::kClsNorm, st);
  switch (H / 256) {
    case 1: embed_ln_kernel<1, FMT><<<B, 256, 0, st>>>(ep); break;
    case 2: embed_ln_kernel<2, FMT><<<B, 256, 0, st>>>(ep); break;
    case 3: embed_ln_kernel<3, FMT><<<B, 256, 0, st>>>(ep); break;
    default: embed_ln_kernel<4, FMT><<<B, 256, 0, st>>>(ep); break;
  }
  ance::prof_end(ance::kClsNorm, st);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  if (e->dbg && M <= e->dbg_tokens) ANCE_CUDA(cudaMemcpyAsync(e->dbg, e->X, static_cast<size_t>(M) * H * 2, cudaMemcpyDeviceToDevice, st));
  AttentionLaunch attn_launch;
  if ((rc = make_attention(attn_launch, e->QKV, e->CTX, M, L, c.heads, e->kbias, varlen ? e->row_lo : nullptr,
                           varlen ? e->row_hi : nullptr, varlen ? e->tile_kv : nullptr))) return rc;
  for (int l = 0; l < c.n_layer; ++l) {
    const LayerDev& d = e->layers[l];
    uint16_t* X_in = ts ? ts->x(l) : e->X;
    uint16_t* QKV = ts ? ts->at(l, ts->lo.qkv) : e->QKV;
    uint16_t* CTX = ts ? ts->at(l, ts->lo.ctx) : e->CTX;
    uint16_t* T1 = ts ? ts->at(l, ts->lo.t1) : e->T;
    uint16_t* X1 = ts ? ts->at(l, ts->lo.x1) : e->X1;
    uint16_t* FF = ts ? ts->at(l, ts->lo.ff) : e->FF;
    uint16_t* T2 = ts ? ts->at(l, ts->lo.t2) : e->T;
    uint16_t* X_out = ts ? ts->x(l + 1) : e->X;
    if (ts && (rc = make_attention(attn_launch, QKV, CTX, M, L, c.heads, ts->kbias(), nullptr, nullptr, nullptr))) return rc;
    if ((rc = linear<FMT>(X_in, H, M, d.wqkv, 3 * H, H, d.bqkv, nullptr, 0, QKV, nullptr, st, ance::kClsGemmQkv))) return rc;
    if ((rc = run_attention<FMT>(attn_launch, st))) return rc;
    // In the last layer only token 0 of every sequence is read downstream (models.py:49,193): run the
    // out-projection, FFN and both LayerNorms on those B rows only (strided TMA views, compact outputs).
    const bool cls_only = (e->prune_last_layer || varlen || ts) && (l == c.n_layer - 1);
    const int Mr = cls_only ? B : M;                                    // rows processed from here on
    const uint16_t *ctx_a = CTX, *res_x = X_in;
    size_t pitch = cls_only ? static_cast<size_t>(L) * H : H;           // row pitch of CTX / X views
    if (cls_only && varlen) {   // the CLS rows sit at seq_row0[b]: gather them into compact [B, H] operands
      ance::ProfScope ps(ance::kClsNorm, st);
      gather_rows16_by_index_kernel<<<B, 96, 0, st>>>(e->CTX, e->seq_row0, B, H, e->cls_ctx);
      gather_rows16_by_index_kernel<<<B, 96, 0, st>>>(e->X, e->seq_row0, B, H, e->cls_x);
      ANCE_CUDA(cudaGetLastError());
      ance::count_launch(2);
      ctx_a = e->cls_ctx; res_x = e->cls_x; pitch = H;
    }
    if ((rc = linear<FMT>(ctx_a, pitch, Mr, d.wo, H, H, d.bo, res_x, 0, T1, nullptr, st, ance::kClsGemmOut, pitch))) return rc;
    if ((rc = layer_norm<FMT>(T1, false, H, Mr, H, d.ln1g, d.ln1b, c.ln_eps, X1, nullptr, st))) return rc;
    if (ts && (rc = linear<FMT>(X1, H, Mr, d.w1, F, H, d.b1, nullptr, 0, ts->at(l, ts->lo.u), nullptr, st, ance::kClsGemmFfn1))) return rc;
    if ((rc = linear<FMT>(X1, H, Mr, d.w1, F, H, d.b1, nullptr, gelu_form(), FF, nullptr, st, ance::kClsGemmFfn1))) return rc;
    if ((rc = linear<FMT>(FF, F, Mr, d.w2, H, F, d.b2, X1, 0, T2, nullptr, st, ance::kClsGemmFfn2))) return rc;
    if ((rc = layer_norm<FMT>(T2, false, H, Mr, H, d.ln2g, d.ln2b, c.ln_eps, X_out, nullptr, st))) return rc;
    if (e->dbg && M <= e->dbg_tokens)  // with cls_only the first B rows hold the CLS rows of the last layer
      ANCE_CUDA(cudaMemcpyAsync(e->dbg + static_cast<size_t>(l + 1) * e->dbg_tokens * H, X_out, static_cast<size_t>(Mr) * H * 2, cudaMemcpyDeviceToDevice, st));
  }
  const size_t cls_pitch = (e->prune_last_layer || varlen || ts) ? static_cast<size_t>(H) : static_cast<size_t>(L) * H;
  const uint16_t* X_last = ts ? ts->x(c.n_layer) : e->X;
  // K7: CLS rows (token 0 of every sequence) -> head
  if (c.has_head) {
    // A = the CLS rows of X ([B, H] compact after the pruned last layer, else row pitch L*H)
    float* head_in = ts ? ts->head_in() : e->head_tmp;
    if ((rc = linear<FMT>(X_last, cls_pitch, B, e->head_w, H, H, e->head_b, nullptr, 0, nullptr, head_in, st))) return rc;
    if ((rc = layer_norm<FMT>(head_in, true, H, B, H, e->head_g, e->head_bt, 1e-5f, nullptr, out_dev, st))) return rc;
  } else {
    ance::ProfScope ps(ance::kClsNorm, st);
    gather_rows_f32_kernel<FMT><<<B, 256, 0, st>>>(X_last, cls_pitch, B, H, out_dev);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
  }
  {
    // overflow of the 16-bit storage format anywhere upstream ends as inf / NaN here (LayerNorm and softmax propagate it)
    ance::ProfScope ps(ance::kClsNorm, st);
    const size_t n = static_cast<size_t>(B) * H;
    check_finite_kernel<<<static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 148)), 256, 0, st>>>(out_dev, n, e->err_flag);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
  }
  return ANCE_OK;
}

}  // namespace

extern "C" int ance_encoder_create(const ance_encoder_config* cfg, const ance_encoder_weights* w, int max_tokens,
                                   ance_encoder_t* out) {
  ANCE_REQUIRE(cfg && w && out, "ance_encoder_create: null argument");
  ANCE_REQUIRE(cfg->hidden % 256 == 0 && cfg->hidden <= 1024, "ance_encoder_create: hidden must be a multiple of 256 (<= 1024), got %d", cfg->hidden);
  ANCE_REQUIRE(cfg->heads * 64 == cfg->hidden, "ance_encoder_create: head_dim must be 64 (hidden %d, heads %d)", cfg->hidden, cfg->heads);
  ANCE_REQUIRE(cfg->ffn % 8 == 0 && cfg->n_layer > 0 && cfg->vocab > 0 && cfg->max_pos > 0, "ance_encoder_create: bad config");
  ANCE_REQUIRE(max_tokens >= 128, "ance_encoder_create: max_tokens must be >= 128");
  ANCE_REQUIRE(!cfg->has_head || (w->head_w && w->head_b && w->head_ln_g && w->head_ln_b), "ance_encoder_create: has_head without head weights");
  ANCE_REQUIRE(cfg->operand_fmt == ANCE_FMT_FP16 || cfg->operand_fmt == ANCE_FMT_BF16, "ance_encoder_create: operand_fmt must be ANCE_FMT_FP16 or ANCE_FMT_BF16, got %d", cfg->operand_fmt);
  int dev = 0;
  if (const int rc = require_sm90(&dev)) return rc;
  ance_encoder* e = new ance_encoder();
  e->cfg = *cfg;
  e->device = dev;
  e->fmt = (cfg->operand_fmt == ANCE_FMT_BF16) ? tc05::kFmtBF16 : tc05::kFmtF16;
  e->max_tokens = (max_tokens + 127) / 128 * 128;
  const size_t H = cfg->hidden, F = cfg->ffn, T = e->max_tokens;
  bool ok = true;
  auto chk = [&](const void* p) { ok = ok && (p != nullptr); };
  chk(e->word = upload_f32(e, w->word_emb, static_cast<size_t>(cfg->vocab) * H));
  chk(e->pos = upload_f32(e, w->pos_emb, static_cast<size_t>(cfg->max_pos) * H));
  chk(e->type = upload_f32(e, w->type_emb, static_cast<size_t>(cfg->type_vocab) * H));
  chk(e->eg = upload_f32(e, w->emb_ln_g, H));
  chk(e->eb = upload_f32(e, w->emb_ln_b, H));
  e->layers.resize(cfg->n_layer);
  for (int l = 0; l < cfg->n_layer && ok; ++l) {
    const ance_layer_weights& lw = w->layers[l];
    LayerDev& d = e->layers[l];
    std::vector<float> wqkv(3 * H * H), bqkv(3 * H);
    memcpy(wqkv.data(), lw.q_w, H * H * 4);
    memcpy(wqkv.data() + H * H, lw.k_w, H * H * 4);
    memcpy(wqkv.data() + 2 * H * H, lw.v_w, H * H * 4);
    memcpy(bqkv.data(), lw.q_b, H * 4);
    memcpy(bqkv.data() + H, lw.k_b, H * 4);
    memcpy(bqkv.data() + 2 * H, lw.v_b, H * 4);
    chk(d.wqkv = upload_16(e, wqkv.data(), wqkv.size()));
    chk(d.bqkv = upload_f32(e, bqkv.data(), bqkv.size()));
    chk(d.wo = upload_16(e, lw.ao_w, H * H));
    chk(d.bo = upload_f32(e, lw.ao_b, H));
    chk(d.ln1g = upload_f32(e, lw.ln1_g, H));
    chk(d.ln1b = upload_f32(e, lw.ln1_b, H));
    chk(d.w1 = upload_16(e, lw.ff1_w, F * H));
    chk(d.b1 = upload_f32(e, lw.ff1_b, F));
    chk(d.w2 = upload_16(e, lw.ff2_w, H * F));
    chk(d.b2 = upload_f32(e, lw.ff2_b, H));
    chk(d.ln2g = upload_f32(e, lw.ln2_g, H));
    chk(d.ln2b = upload_f32(e, lw.ln2_b, H));
  }
  if (cfg->has_head && ok) {
    chk(e->head_w = upload_16(e, w->head_w, H * H));
    chk(e->head_b = upload_f32(e, w->head_b, H));
    chk(e->head_g = upload_f32(e, w->head_ln_g, H));
    chk(e->head_bt = upload_f32(e, w->head_ln_b, H));
  }
  chk(e->X = dev_alloc<uint16_t>(e, T * H));
  chk(e->QKV = dev_alloc<uint16_t>(e, T * 3 * H));
  chk(e->CTX = dev_alloc<uint16_t>(e, T * H));
  chk(e->T = dev_alloc<uint16_t>(e, T * H));
  chk(e->X1 = dev_alloc<uint16_t>(e, T * H));
  chk(e->FF = dev_alloc<uint16_t>(e, T * F));
  chk(e->kbias = dev_alloc<float>(e, T));
  chk(e->cls_ctx = dev_alloc<uint16_t>(e, T / 16 * H));
  chk(e->cls_x = dev_alloc<uint16_t>(e, T / 16 * H));
  chk(e->seq_row0 = dev_alloc<int32_t>(e, T / 16));
  chk(e->row_lo = dev_alloc<int32_t>(e, T));
  chk(e->row_hi = dev_alloc<int32_t>(e, T));
  chk(e->tile_kv = dev_alloc<int2>(e, T / attn::kTile));
  chk(e->head_tmp = dev_alloc<float>(e, T / 16 * H));
  chk(e->err_flag = dev_alloc<int>(e, 1));
  if (!ok || cudaGetLastError() != cudaSuccess) {
    ance::set_error("ance_encoder_create: device allocation / upload failed (max_tokens %d)", max_tokens);
    ance_encoder_destroy(e);
    return ANCE_ERR_NOMEM;
  }
  cudaMemset(e->err_flag, 0, sizeof(int));
  const int rc = (e->fmt == tc05::kFmtBF16) ? set_attention_attrs<tc05::kFmtBF16>() : set_attention_attrs<tc05::kFmtF16>();
  if (rc) {
    ance_encoder_destroy(e);
    return rc;
  }
  *out = e;
  return ANCE_OK;
}

extern "C" int ance_encoder_destroy(ance_encoder_t e) {
  if (!e) return ANCE_OK;
  for (void* p : e->allocs) cudaFree(p);
  if (e->bwd_scratch) cudaFree(e->bwd_scratch);
  if (e->refresh_dev) cudaFree(e->refresh_dev);
  delete e;
  return ANCE_OK;
}

extern "C" int ance_encoder_forward(ance_encoder_t e, const int32_t* ids_dev, const int32_t* lens_dev,
                                    const uint8_t* mask_dev, int B, int L, float* out_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_forward: null handle");
  ANCE_REQUIRE(ids_dev && out_dev, "ance_encoder_forward: null buffer");
  ANCE_REQUIRE((lens_dev != nullptr) != (mask_dev != nullptr), "ance_encoder_forward: pass exactly one of lens_dev / mask_dev");
  ANCE_REQUIRE(B > 0 && L > 0, "ance_encoder_forward: empty batch");
  ANCE_REQUIRE(L <= 512 && ((L % 128 == 0) || (128 % L == 0 && L >= 8)), "ance_encoder_forward: L = %d unsupported (need a multiple of 128 up to 512, or a divisor of 128)", L);
  const ance_encoder_config& c = e->cfg;
  ANCE_REQUIRE(L + (c.arch == ANCE_ARCH_ROBERTA ? c.pad_id + 1 : 0) <= c.max_pos, "ance_encoder_forward: L = %d exceeds max_position_embeddings %d", L, c.max_pos);
  const long long tokens = static_cast<long long>(B) * L;
  ANCE_REQUIRE(tokens <= e->max_tokens, "ance_encoder_forward: %lld tokens exceed max_tokens %d", tokens, e->max_tokens);
  ANCE_REQUIRE(B <= e->max_tokens / 16, "ance_encoder_forward: batch %d too large for the head buffer", B);
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == e->device, "ance_encoder_forward: the handle belongs to device %d but device %d is current", e->device, dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (e->fmt == tc05::kFmtBF16) return forward_impl<tc05::kFmtBF16>(e, ids_dev, lens_dev, mask_dev, B, L, out_dev, st);
  return forward_impl<tc05::kFmtF16>(e, ids_dev, lens_dev, mask_dev, B, L, out_dev, st);
}

// ------------------------------------------------------------------------------------------------
// training: forward with saved activations, backward, in-place weight refresh
// ------------------------------------------------------------------------------------------------
namespace {

constexpr uint32_t kBF = tc05::kFmtBF16;   // every backward GEMM runs on bf16 operands (gradients can underflow fp16)

unsigned ew_grid(size_t n) { return static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 8192)); }

// dst [C, dst_ld] bf16 = src[R, C]^T (kSrc 0 fp16, 1 bf16, 2 fp32), columns R .. dst_ld - 1 zero
template <int kSrc>
int transpose_bf16(const void* src, size_t src_ld, int R, int C, uint16_t* dst, size_t dst_ld, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((dst_ld + 31) / 32), static_cast<unsigned>((C + 31) / 32));
  bwd::transpose_bf16_kernel<kSrc><<<grid, dim3(32, 8), 0, st>>>(src, src_ld, R, C, dst, dst_ld);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

template <uint32_t FMT>
constexpr int src_code() { return FMT == tc05::kFmtBF16 ? 1 : 0; }

int to_bf16(const float* a, uint16_t* o, size_t n, cudaStream_t st) {
  bwd::f32_to_bf16_kernel<<<ew_grid(n), 256, 0, st>>>(a, o, n);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

int add_rows(float* dst, size_t dst_row_stride, const float* src, int rows, int H, cudaStream_t st) {
  bwd::add_rows_kernel<<<ew_grid(static_cast<size_t>(rows) * H), 256, 0, st>>>(dst, dst_row_stride, src, rows, H);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

// column sums of fp32 a [rows, N] -> o0 / o1 / o2 (segments of `seg` columns), deterministic
int colsum(const float* a, int rows, int N, float* part, int seg, float* o0, float* o1, float* o2, cudaStream_t st) {
  int chunks = std::min(rows, bwd::kColsumChunks);
  const int per = (rows + chunks - 1) / chunks;
  chunks = (rows + per - 1) / per;
  bwd::colsum_partial_kernel<<<dim3((N + 255) / 256, chunks), 256, 0, st>>>(a, rows, N, per, part);
  bwd::colsum_final_kernel<<<(N + 255) / 256, 256, 0, st>>>(part, chunks, N, seg, o0, o1, o2);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(2);
  return ANCE_OK;
}

// LayerNorm backward of `rows` rows + dgamma / dbeta / dbias (any of the three may be null); part: scratch of
// kLnBwdMaxBlocks * 3H floats
template <uint32_t FMT>
int ln_bwd(const void* x, bool in_f32, size_t x_ld, int rows, int H, const float* gamma, float eps, const float* dy,
           float* dx, float* part, float* dgamma, float* dbeta, float* dbias, cudaStream_t st) {
  const int blocks = std::min((rows + 7) / 8, bwd::kLnBwdMaxBlocks);
  ance::ProfScope ps(ance::kClsNorm, st);
#define LNB_CASE(NV_)                                                                                                  \
  if (in_f32) bwd::ln_bwd_kernel<NV_, true, FMT><<<blocks, 256, 0, st>>>(x, x_ld, rows, H, gamma, eps, dy, dx, part);   \
  else bwd::ln_bwd_kernel<NV_, false, FMT><<<blocks, 256, 0, st>>>(x, x_ld, rows, H, gamma, eps, dy, dx, part)
  switch (H / 256) {
    case 1: LNB_CASE(1); break;
    case 2: LNB_CASE(2); break;
    case 3: LNB_CASE(3); break;
    case 4: LNB_CASE(4); break;
    default: ance::set_error("encoder backward: hidden size %d unsupported", H); return ANCE_ERR_UNSUPPORTED;
  }
#undef LNB_CASE
  bwd::colsum_final_kernel<<<(3 * H + 255) / 256, 256, 0, st>>>(part, blocks, 3 * H, H, dgamma, dbeta, dbias);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(2);
  return ANCE_OK;
}

template <uint32_t FMT>
int attn_bwd(const uint16_t* qkv, const float* kbias, const uint16_t* dout, bool cls_only, float* dqkv, int B, int L,
             int heads, cudaStream_t st) {
  const size_t smem = bwd::attn_bwd_smem(L);
  ANCE_CUDA(cudaFuncSetAttribute(bwd::attn_bwd_kernel<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bwd::attn_bwd_smem(attn::kTile))));
  ance::ProfScope ps(ance::kClsAttn, st);
  bwd::attn_bwd_kernel<FMT><<<dim3(B, heads), 256, smem, st>>>(qkv, kbias, dout, cls_only ? 1 : 0, dqkv, L, heads, kLog2e / 8.0f);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

// bf16 W^T copies of every linear weight (dgrad operands), rebuilt from the 16-bit weights after a change
template <uint32_t FMT>
int ensure_wt(ance_encoder* e, cudaStream_t st) {
  const ance_encoder_config& c = e->cfg;
  const size_t H = c.hidden, F = c.ffn;
  if (e->wt.empty()) {
    std::vector<ance_encoder::LayerT> wt(c.n_layer);
    bool ok = true;
    for (auto& t : wt) {
      ok = ok && (t.wqkv = dev_alloc<uint16_t>(e, 3 * H * H)) && (t.wo = dev_alloc<uint16_t>(e, H * H)) &&
           (t.w1 = dev_alloc<uint16_t>(e, F * H)) && (t.w2 = dev_alloc<uint16_t>(e, H * F));
    }
    if (c.has_head) ok = ok && (e->head_wt = dev_alloc<uint16_t>(e, H * H));
    if (!ok) {
      ance::set_error("encoder backward: allocating the transposed weights failed");
      return ANCE_ERR_NOMEM;
    }
    e->wt = wt;
    e->wt_stale = true;
  }
  if (!e->wt_stale) return ANCE_OK;
  constexpr int S = src_code<FMT>();
  int rc;
  for (int l = 0; l < c.n_layer; ++l) {
    const LayerDev& d = e->layers[l];
    const ance_encoder::LayerT& t = e->wt[l];
    if ((rc = transpose_bf16<S>(d.wqkv, H, 3 * H, H, t.wqkv, 3 * H, st))) return rc;
    if ((rc = transpose_bf16<S>(d.wo, H, H, H, t.wo, H, st))) return rc;
    if ((rc = transpose_bf16<S>(d.w1, H, F, H, t.w1, F, st))) return rc;
    if ((rc = transpose_bf16<S>(d.w2, F, H, F, t.w2, H, st))) return rc;
  }
  if (c.has_head && (rc = transpose_bf16<S>(e->head_w, H, H, H, e->head_wt, H, st))) return rc;
  e->wt_stale = false;
  return ANCE_OK;
}

struct BwdScratch {
  float *G, *dT, *dA, *dX1, *part;
  uint16_t *A16, *Gt, *Xt, *dCTX;
  int32_t* pos;
};

int ensure_scratch(ance_encoder* e, int M, BwdScratch& s) {
  const size_t H = e->cfg.hidden, F = e->cfg.ffn, N = std::max(3 * H, F), Mp = (M + 7) / 8 * 8;
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t part = std::max(static_cast<size_t>(bwd::kLnBwdMaxBlocks) * 3 * H, static_cast<size_t>(bwd::kColsumChunks) * N);
  const size_t sz[10] = {up(M * H * 4), up(M * H * 4), up(M * N * 4), up(M * H * 4), up(part * 4),
                         up(M * N * 2), up(N * Mp * 2), up(N * Mp * 2), up(M * H * 2), up(static_cast<size_t>(M) * 4)};
  size_t total = 0;
  for (size_t x : sz) total += x;
  if (total > e->bwd_scratch_bytes) {
    if (e->bwd_scratch) cudaFree(e->bwd_scratch);
    e->bwd_scratch = nullptr;
    e->bwd_scratch_bytes = 0;
    if (cudaMalloc(&e->bwd_scratch, total) != cudaSuccess) {
      e->bwd_scratch = nullptr;
      ance::set_error("encoder backward: allocating %zu bytes of scratch failed", total);
      return ANCE_ERR_NOMEM;
    }
    e->bwd_scratch_bytes = total;
  }
  uint8_t* p = reinterpret_cast<uint8_t*>(e->bwd_scratch);
  void* q[10];
  for (int i = 0; i < 10; ++i) { q[i] = p; p += sz[i]; }
  s.G = static_cast<float*>(q[0]); s.dT = static_cast<float*>(q[1]); s.dA = static_cast<float*>(q[2]);
  s.dX1 = static_cast<float*>(q[3]); s.part = static_cast<float*>(q[4]);
  s.A16 = static_cast<uint16_t*>(q[5]); s.Gt = static_cast<uint16_t*>(q[6]); s.Xt = static_cast<uint16_t*>(q[7]);
  s.dCTX = static_cast<uint16_t*>(q[8]); s.pos = static_cast<int32_t*>(q[9]);
  return ANCE_OK;
}

// C32 [N_out, K_in] = dY^T X over `rows` tokens: A = dY^T [N_out, rows_p] and W = X^T [K_in, rows_p] (bf16, zero columns
// past `rows`, so K = rows_p is exact)
int wgrad(const uint16_t* dYt, int n_out, const uint16_t* Xt, int k_in, int rows_p, float* C32, cudaStream_t st) {
  return linear<kBF>(dYt, rows_p, n_out, Xt, k_in, rows_p, nullptr, nullptr, 0, nullptr, C32, st);
}

template <uint32_t FMT>
int backward_impl(ance_encoder* e, int B, int L, const float* d_out, uint8_t* ws, const ance_encoder_grads* g,
                  cudaStream_t st) {
  const ance_encoder_config& c = e->cfg;
  const int H = c.hidden, F = c.ffn, M = B * L, Mp = (M + 7) / 8 * 8, NL = c.n_layer;
  constexpr int S = src_code<FMT>();
  TrainSave ts{ws, train_layout(c, B, L), NL};
  BwdScratch s;
  int rc;
  if ((rc = ensure_wt<FMT>(e, st))) return rc;
  if ((rc = ensure_scratch(e, M, s))) return rc;
  const int Bp = (B + 7) / 8 * 8;
  // head: out = LN(X_cls Wh^T + bh) -> s.G = d X_cls [B, H]
  if (c.has_head) {
    if ((rc = ln_bwd<FMT>(ts.head_in(), true, H, B, H, e->head_g, 1e-5f, d_out, s.dT, s.part, g->head_ln_g, g->head_ln_b, g->head_b, st))) return rc;
    if ((rc = to_bf16(s.dT, s.A16, static_cast<size_t>(B) * H, st))) return rc;
    if ((rc = transpose_bf16<2>(s.dT, H, B, H, s.Gt, Bp, st))) return rc;
    if ((rc = transpose_bf16<S>(ts.x(NL), H, B, H, s.Xt, Bp, st))) return rc;
    if ((rc = wgrad(s.Gt, H, s.Xt, H, Bp, g->head_w, st))) return rc;
    if ((rc = linear<kBF>(s.A16, H, B, e->head_wt, H, H, nullptr, nullptr, 0, nullptr, s.G, st))) return rc;
  } else {
    ANCE_CUDA(cudaMemcpyAsync(s.G, d_out, static_cast<size_t>(B) * H * 4, cudaMemcpyDeviceToDevice, st));
  }
  for (int l = NL - 1; l >= 0; --l) {
    const LayerDev& d = e->layers[l];
    const ance_encoder::LayerT& wt = e->wt[l];
    const ance_layer_grads& lg = g->layers[l];
    const bool last = l == NL - 1;
    const int Mr = last ? B : M, Mrp = (Mr + 7) / 8 * 8;
    // s.G = d X_out [Mr, H].  LN2: T2 = FF W2^T + b2 + X1
    if ((rc = ln_bwd<FMT>(ts.at(l, ts.lo.t2), false, H, Mr, H, d.ln2g, c.ln_eps, s.G, s.dT, s.part, lg.ln2_g, lg.ln2_b, lg.ff2_b, st))) return rc;
    if ((rc = to_bf16(s.dT, s.A16, static_cast<size_t>(Mr) * H, st))) return rc;
    if ((rc = transpose_bf16<2>(s.dT, H, Mr, H, s.Gt, Mrp, st))) return rc;
    if ((rc = transpose_bf16<S>(ts.at(l, ts.lo.ff), F, Mr, F, s.Xt, Mrp, st))) return rc;
    if ((rc = wgrad(s.Gt, H, s.Xt, F, Mrp, lg.ff2_w, st))) return rc;
    if ((rc = linear<kBF>(s.A16, H, Mr, wt.w2, F, H, nullptr, nullptr, 0, nullptr, s.dA, st))) return rc;   // d FF
    {
      const size_t n = static_cast<size_t>(Mr) * F;
      bwd::gelu_bwd_kernel<FMT><<<ew_grid(n), 256, 0, st>>>(ts.at(l, ts.lo.u), s.dA, n);   // d U
      ANCE_CUDA(cudaGetLastError());
      ance::count_launch(1);
    }
    if ((rc = colsum(s.dA, Mr, F, s.part, F, lg.ff1_b, nullptr, nullptr, st))) return rc;
    if ((rc = to_bf16(s.dA, s.A16, static_cast<size_t>(Mr) * F, st))) return rc;
    if ((rc = transpose_bf16<2>(s.dA, F, Mr, F, s.Gt, Mrp, st))) return rc;
    if ((rc = transpose_bf16<S>(ts.at(l, ts.lo.x1), H, Mr, H, s.Xt, Mrp, st))) return rc;
    if ((rc = wgrad(s.Gt, F, s.Xt, H, Mrp, lg.ff1_w, st))) return rc;
    if ((rc = linear<kBF>(s.A16, F, Mr, wt.w1, H, F, nullptr, nullptr, 0, nullptr, s.dX1, st))) return rc;   // d X1 (FFN)
    if ((rc = add_rows(s.dX1, 1, s.dT, Mr, H, st))) return rc;                                              // + residual
    // LN1: T1 = CTX Wo^T + bo + X_in
    if ((rc = ln_bwd<FMT>(ts.at(l, ts.lo.t1), false, H, Mr, H, d.ln1g, c.ln_eps, s.dX1, s.dT, s.part, lg.ln1_g, lg.ln1_b, lg.ao_b, st))) return rc;
    if ((rc = to_bf16(s.dT, s.A16, static_cast<size_t>(Mr) * H, st))) return rc;
    if ((rc = transpose_bf16<2>(s.dT, H, Mr, H, s.Gt, Mrp, st))) return rc;
    if ((rc = transpose_bf16<S>(ts.at(l, ts.lo.ctx), last ? static_cast<size_t>(L) * H : H, Mr, H, s.Xt, Mrp, st))) return rc;
    if ((rc = wgrad(s.Gt, H, s.Xt, H, Mrp, lg.ao_w, st))) return rc;
    if ((rc = linear<kBF>(s.A16, H, Mr, wt.wo, H, H, nullptr, nullptr, 0, s.dCTX, nullptr, st))) return rc;  // d CTX (bf16)
    // attention -> d QKV [M, 3H]
    if ((rc = attn_bwd<FMT>(ts.at(l, ts.lo.qkv), ts.kbias(), s.dCTX, last, s.dA, B, L, c.heads, st))) return rc;
    if ((rc = colsum(s.dA, M, 3 * H, s.part, H, lg.q_b, lg.k_b, lg.v_b, st))) return rc;
    if ((rc = to_bf16(s.dA, s.A16, static_cast<size_t>(M) * 3 * H, st))) return rc;
    if ((rc = transpose_bf16<2>(s.dA, 3 * H, M, 3 * H, s.Gt, Mp, st))) return rc;
    if ((rc = transpose_bf16<S>(ts.x(l), H, M, H, s.Xt, Mp, st))) return rc;
    float* const wq[3] = {lg.q_w, lg.k_w, lg.v_w};
    for (int p = 0; p < 3; ++p)
      if ((rc = wgrad(s.Gt + static_cast<size_t>(p) * H * Mp, H, s.Xt, H, Mp, wq[p], st))) return rc;
    if ((rc = linear<kBF>(s.A16, 3 * H, M, wt.wqkv, H, 3 * H, nullptr, nullptr, 0, nullptr, s.G, st))) return rc;   // d X_in
    if ((rc = add_rows(s.G, last ? L : 1, s.dT, Mr, H, st))) return rc;   // + residual (the CLS rows in the last layer)
  }
  // embeddings: X0 = LN((word[id] + pos[p]) + type[0])
  {
    ance::ProfScope ps(ance::kClsNorm, st);
    bwd::embed_sum_kernel<<<B, 256, 0, st>>>(ts.ids(), L, H, c.arch == ANCE_ARCH_ROBERTA, c.pad_id, c.vocab, c.max_pos,
                                             e->word, e->pos, e->type, s.dA, s.pos);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
  }
  ANCE_CUDA(cudaMemsetAsync(g->word_emb, 0, static_cast<size_t>(c.vocab) * H * 4, st));
  ANCE_CUDA(cudaMemsetAsync(g->pos_emb, 0, static_cast<size_t>(c.max_pos) * H * 4, st));
  ANCE_CUDA(cudaMemsetAsync(g->type_emb, 0, static_cast<size_t>(c.type_vocab) * H * 4, st));
  if ((rc = ln_bwd<FMT>(s.dA, true, H, M, H, e->eg, c.ln_eps, s.G, s.dT, s.part, g->emb_ln_g, g->emb_ln_b, g->type_emb, st))) return rc;
  {
    ance::ProfScope ps(ance::kClsNorm, st);
    bwd::embed_scatter_kernel<<<M, 256, 0, st>>>(ts.ids(), s.pos, s.dT, M, H, c.arch == ANCE_ARCH_ROBERTA, c.pad_id, c.vocab,
                                                 g->word_emb, g->pos_emb);
    ANCE_CUDA(cudaGetLastError());
    ance::count_launch(1);
  }
  return ANCE_OK;
}

// One launch converts every parameter into the handle: a table of (source, destination, count, kind) pieces of at most
// bwd::kRefreshChunk elements, one block each.  The table is re-uploaded only when a pointer changed.
template <uint32_t FMT>
int update_weights_impl(ance_encoder* e, const ance_encoder_weights* w, cudaStream_t st) {
  const ance_encoder_config& c = e->cfg;
  const size_t H = c.hidden, F = c.ffn;
  std::vector<bwd::RefreshPiece> t;
  auto add = [&](const float* src, void* dst, size_t n, uint32_t to16) {
    for (size_t o = 0; o < n; o += bwd::kRefreshChunk) {
      bwd::RefreshPiece r;
      r.src = src + o;
      r.dst = to16 ? static_cast<void*>(static_cast<uint16_t*>(dst) + o) : static_cast<void*>(static_cast<float*>(dst) + o);
      r.n = static_cast<uint32_t>(std::min<size_t>(bwd::kRefreshChunk, n - o));
      r.to16 = to16;
      t.push_back(r);
    }
  };
  add(w->word_emb, e->word, static_cast<size_t>(c.vocab) * H, 0);
  add(w->pos_emb, e->pos, static_cast<size_t>(c.max_pos) * H, 0);
  add(w->type_emb, e->type, static_cast<size_t>(c.type_vocab) * H, 0);
  add(w->emb_ln_g, e->eg, H, 0);
  add(w->emb_ln_b, e->eb, H, 0);
  for (int l = 0; l < c.n_layer; ++l) {
    const ance_layer_weights& lw = w->layers[l];
    const LayerDev& d = e->layers[l];
    add(lw.q_w, d.wqkv, H * H, 1);
    add(lw.k_w, d.wqkv + H * H, H * H, 1);
    add(lw.v_w, d.wqkv + 2 * H * H, H * H, 1);
    add(lw.q_b, d.bqkv, H, 0);
    add(lw.k_b, d.bqkv + H, H, 0);
    add(lw.v_b, d.bqkv + 2 * H, H, 0);
    add(lw.ao_w, d.wo, H * H, 1);
    add(lw.ao_b, d.bo, H, 0);
    add(lw.ln1_g, d.ln1g, H, 0);
    add(lw.ln1_b, d.ln1b, H, 0);
    add(lw.ff1_w, d.w1, F * H, 1);
    add(lw.ff1_b, d.b1, F, 0);
    add(lw.ff2_w, d.w2, H * F, 1);
    add(lw.ff2_b, d.b2, H, 0);
    add(lw.ln2_g, d.ln2g, H, 0);
    add(lw.ln2_b, d.ln2b, H, 0);
  }
  if (c.has_head) {
    add(w->head_w, e->head_w, H * H, 1);
    add(w->head_b, e->head_b, H, 0);
    add(w->head_ln_g, e->head_g, H, 0);
    add(w->head_ln_b, e->head_bt, H, 0);
  }
  const size_t bytes = t.size() * sizeof(bwd::RefreshPiece);
  const bool same = e->refresh_table.size() == t.size() && memcmp(e->refresh_table.data(), t.data(), bytes) == 0;
  if (!same) {
    if (t.size() > e->refresh_cap) {   // grows once; the old table is freed after the work queued before it
      if (e->refresh_dev) ANCE_CUDA(cudaFreeAsync(e->refresh_dev, st));
      e->refresh_dev = nullptr;
      e->refresh_cap = 0;
      ANCE_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&e->refresh_dev), bytes, st));
      e->refresh_cap = t.size();
    }
    e->refresh_table = t;   // kept alive: the pageable copy below reads it
    ANCE_CUDA(cudaMemcpyAsync(e->refresh_dev, e->refresh_table.data(), bytes, cudaMemcpyHostToDevice, st));
  }
  bwd::refresh_kernel<FMT><<<static_cast<unsigned>(t.size()), 256, 0, st>>>(e->refresh_dev);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  e->wt_stale = true;
  return ANCE_OK;
}

// ance_encoder_grads is ance_encoder_weights with writable pointers: the same checks serve both
static_assert(sizeof(ance_layer_grads) == sizeof(ance_layer_weights) && sizeof(ance_encoder_grads) == sizeof(ance_encoder_weights),
              "gradient and weight structs must share one layout");

// every pointer the config needs is non-null (and, with `aligned`, 16-byte aligned: the kernels use 16-byte accesses)
bool weights_complete(const ance_encoder_config& c, const ance_encoder_weights* w, bool aligned = false) {
  auto ok = [&](const void* q) { return q && (!aligned || (reinterpret_cast<uintptr_t>(q) & 15u) == 0); };
  if (!ok(w->word_emb) || !ok(w->pos_emb) || !ok(w->type_emb) || !ok(w->emb_ln_g) || !ok(w->emb_ln_b) || !w->layers) return false;
  for (int l = 0; l < c.n_layer; ++l) {
    const ance_layer_weights& x = w->layers[l];
    const float* const p[16] = {x.q_w, x.q_b, x.k_w, x.k_b, x.v_w, x.v_b, x.ao_w, x.ao_b, x.ln1_g, x.ln1_b,
                                x.ff1_w, x.ff1_b, x.ff2_w, x.ff2_b, x.ln2_g, x.ln2_b};
    for (const float* q : p)
      if (!ok(q)) return false;
  }
  return !c.has_head || (ok(w->head_w) && ok(w->head_b) && ok(w->head_ln_g) && ok(w->head_ln_b));
}

}  // namespace

extern "C" int ance_encoder_train_workspace(ance_encoder_t e, int B, int L, size_t* bytes) {
  ANCE_REQUIRE(e != nullptr && bytes != nullptr, "ance_encoder_train_workspace: null argument");
  ANCE_REQUIRE(B > 0 && L > 0, "ance_encoder_train_workspace: empty batch");
  if (L > attn::kTile) {
    ance::set_error("ance_encoder_train_workspace: L = %d; the backward covers sequences of up to 128 tokens", L);
    return ANCE_ERR_UNSUPPORTED;
  }
  *bytes = train_layout(e->cfg, B, L).total;
  return ANCE_OK;
}

extern "C" int ance_encoder_forward_train(ance_encoder_t e, const int32_t* ids_dev, const int32_t* lens_dev,
                                          const uint8_t* mask_dev, int B, int L, void* ws_dev, float* out_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_forward_train: null handle");
  ANCE_REQUIRE(ids_dev && out_dev && ws_dev, "ance_encoder_forward_train: null buffer");
  ANCE_REQUIRE((lens_dev != nullptr) != (mask_dev != nullptr), "ance_encoder_forward_train: pass exactly one of lens_dev / mask_dev");
  ANCE_REQUIRE(B > 0 && L > 0, "ance_encoder_forward_train: empty batch");
  if (L > attn::kTile) {
    ance::set_error("ance_encoder_forward_train: L = %d; the backward covers sequences of up to 128 tokens", L);
    return ANCE_ERR_UNSUPPORTED;
  }
  ANCE_REQUIRE(128 % L == 0 && L >= 8, "ance_encoder_forward_train: L = %d unsupported (need a divisor of 128, >= 8)", L);
  ANCE_REQUIRE((reinterpret_cast<uintptr_t>(ws_dev) & 255u) == 0, "ance_encoder_forward_train: the workspace must be 256-byte aligned");
  const ance_encoder_config& c = e->cfg;
  ANCE_REQUIRE(L + (c.arch == ANCE_ARCH_ROBERTA ? c.pad_id + 1 : 0) <= c.max_pos, "ance_encoder_forward_train: L = %d exceeds max_position_embeddings %d", L, c.max_pos);
  const long long tokens = static_cast<long long>(B) * L;
  ANCE_REQUIRE(tokens <= e->max_tokens, "ance_encoder_forward_train: %lld tokens exceed max_tokens %d", tokens, e->max_tokens);
  ANCE_REQUIRE(B <= e->max_tokens / 16, "ance_encoder_forward_train: batch %d too large for the head buffer", B);
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == e->device, "ance_encoder_forward_train: the handle belongs to device %d but device %d is current", e->device, dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const TrainSave ts{reinterpret_cast<uint8_t*>(ws_dev), train_layout(c, B, L), c.n_layer};
  e->train_shapes[ws_dev] = make_int2(B, L);
  if (e->fmt == tc05::kFmtBF16) return forward_impl<tc05::kFmtBF16>(e, ids_dev, lens_dev, mask_dev, B, L, out_dev, st, 0, &ts);
  return forward_impl<tc05::kFmtF16>(e, ids_dev, lens_dev, mask_dev, B, L, out_dev, st, 0, &ts);
}

extern "C" int ance_encoder_backward(ance_encoder_t e, const float* d_out_dev, void* ws_dev, const ance_encoder_grads* g,
                                     void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_backward: null handle");
  ANCE_REQUIRE(d_out_dev && ws_dev && g, "ance_encoder_backward: null argument");
  ANCE_REQUIRE((reinterpret_cast<uintptr_t>(d_out_dev) & 15u) == 0, "ance_encoder_backward: d_out must be 16-byte aligned");
  const auto it = e->train_shapes.find(ws_dev);
  ANCE_REQUIRE(it != e->train_shapes.end(), "ance_encoder_backward: the workspace was not filled by ance_encoder_forward_train on "
               "this handle, or its backward has already run");
  const ance_encoder_config& c = e->cfg;
  ANCE_REQUIRE(weights_complete(c, reinterpret_cast<const ance_encoder_weights*>(g), true),
               "ance_encoder_backward: a gradient pointer is null or not 16-byte aligned");
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == e->device, "ance_encoder_backward: the handle belongs to device %d but device %d is current", e->device, dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* ws = reinterpret_cast<uint8_t*>(ws_dev);
  const int2 shape = it->second;
  e->train_shapes.erase(it);   // one backward per forward_train: the record cannot outlive the caller's workspace
  if (e->fmt == tc05::kFmtBF16) return backward_impl<tc05::kFmtBF16>(e, shape.x, shape.y, d_out_dev, ws, g, st);
  return backward_impl<tc05::kFmtF16>(e, shape.x, shape.y, d_out_dev, ws, g, st);
}

extern "C" int ance_encoder_update_weights(ance_encoder_t e, const ance_encoder_weights* w_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr && w_dev != nullptr, "ance_encoder_update_weights: null argument");
  ANCE_REQUIRE(weights_complete(e->cfg, w_dev), "ance_encoder_update_weights: a weight pointer is null");
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == e->device, "ance_encoder_update_weights: the handle belongs to device %d but device %d is current", e->device, dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (e->fmt == tc05::kFmtBF16) return update_weights_impl<tc05::kFmtBF16>(e, w_dev, st);
  return update_weights_impl<tc05::kFmtF16>(e, w_dev, st);
}

// ------------------------------------------------------------------------------------------------
// variable-length forward: whole sequences packed into 128-row attention tiles
// ------------------------------------------------------------------------------------------------
namespace {

struct PackPlan {
  std::vector<int32_t> row0;     // [placed] first packed row of each sequence
  std::vector<int32_t> lo, hi;   // [n_tiles * 128] own-sequence key range of every packed row (absolute rows)
  std::vector<int2> tile_kv;     // [n_tiles] (first key row, number of 128-key blocks) of the tile's attention items
  int n_tiles = 0;
};

// Plans sequences first .. (in order) into at most cap_tiles tiles of 128 rows; stops at the first sequence that fits
// nowhere, or at max_seqs.  Returns the number of sequences placed (a sequence never crosses a chunk of work).
//
// Sequences of <= 128 tokens: online best-fit — every sequence goes to the fullest tile that still has room for it (all
// tiles of the chunk stay open, so this packs almost as well as an offline pass); no sequence straddles a tile.
// align: every such sequence starts at a multiple of `align` rows of its tile (its slot is padded up to a multiple).  With
// align = 16 — the K step of a 16-bit wgmma — the P*V accumulation and the softmax row sum of a sequence group their
// terms exactly as they do at offset 0, so its embedding does not depend on what else is in the tile and equals the dense
// forward's bit for bit; align = 1 packs ~12 % more real tokens per tile.
//
// L > 128 (long = more than 128 tokens):
//   align = 16 (exact): a long sequence starts on a tile boundary and fills ceil(len / 128) consecutive tiles, so its key
//     blocks are the dense kernel's.  Its rows are padded up to a multiple of 32 with its own padding tokens: the softmax
//     warp that holds its last rows then holds the same 32 query rows as in the dense forward (the warp votes on a
//     re-scaling pass together).  Shorter sequences take the best-fit rule above, also in the free rows of a long
//     sequence's last tile.  Every embedding is bit-identical to the dense forward at the same L.
//   align = 1 (densest): every sequence starts where the previous one ends; an attention item then reads the keys of every
//     sequence its tile touches, possibly more than 4 blocks.
int pack_chunk(const int32_t* lens, int first, int B, int L, int cap_tiles, int max_seqs, int align, PackPlan& plan) {
  constexpr int T = attn::kTile;
  const bool long_rules = L > T;
  std::vector<int> used;            // rows used per tile
  std::vector<int> head(T + 1, -1); // head[f] = a tile with exactly f free rows (intrusive lists through next[])
  std::vector<int> next;
  std::vector<int> rows;            // rows computed per placed sequence
  plan.row0.clear();
  auto push = [&](int tile) { const int f = T - used[tile]; next[tile] = head[f]; head[f] = tile; };
  int placed = 0, cursor = 0;
  for (int b = first; b < B && placed < max_seqs; ++b) {
    const int len = lens[b];
    if (long_rules && align == 1) {   // densest: contiguous
      if (cursor + len > cap_tiles * T) break;
      plan.row0.push_back(cursor);
      rows.push_back(len);
      cursor += len;
      ++placed;
      continue;
    }
    if (long_rules && len > T) {      // exact, long: fresh tiles
      const int n = (len + T - 1) / T;
      if (static_cast<int>(used.size()) + n > cap_tiles) break;
      const int r = std::min((len + 31) / 32 * 32, L);
      const int t0 = static_cast<int>(used.size());
      for (int k = 0; k < n; ++k) {
        used.push_back(std::min(T, r - k * T));
        next.push_back(-1);
      }
      if (used.back() < T) push(t0 + n - 1);
      plan.row0.push_back(t0 * T);
      rows.push_back(r);
      ++placed;
      continue;
    }
    const int slot = (len + align - 1) / align * align;   // rows of the slot
    int tile = -1;
    for (int f = slot; f <= T; ++f)   // smallest free space that fits = fullest tile
      if (head[f] >= 0) { tile = head[f]; head[f] = next[tile]; break; }
    if (tile < 0) {
      if (static_cast<int>(used.size()) >= cap_tiles) break;
      tile = static_cast<int>(used.size());
      used.push_back(0);
      next.push_back(-1);
    }
    plan.row0.push_back(tile * T + used[tile]);
    rows.push_back(len);
    used[tile] += slot;
    if (used[tile] < T) push(tile);
    ++placed;
  }
  const int n_tiles = (long_rules && align == 1) ? (cursor + T - 1) / T : static_cast<int>(used.size());
  plan.lo.resize(static_cast<size_t>(n_tiles) * T);
  plan.hi.resize(static_cast<size_t>(n_tiles) * T);
  for (int r = 0; r < n_tiles * T; ++r) {   // default: a row that belongs to no sequence attends to itself
    plan.lo[r] = r;
    plan.hi[r] = r + 1;
  }
  for (int i = 0; i < placed; ++i) {
    const int r0 = plan.row0[i], len = lens[first + i];
    for (int t = 0; t < rows[i]; ++t) {
      plan.lo[r0 + t] = r0;
      plan.hi[r0 + t] = r0 + len;
    }
  }
  plan.tile_kv.resize(n_tiles);
  for (int t = 0; t < n_tiles; ++t) {   // keys of a tile: from the smallest own-sequence start to the largest end
    int kv0 = plan.lo[t * T], kv1 = plan.hi[t * T];
    for (int r = t * T; r < (t + 1) * T; ++r) {
      kv0 = std::min(kv0, plan.lo[r]);
      kv1 = std::max(kv1, plan.hi[r]);
    }
    plan.tile_kv[t] = make_int2(kv0, (kv1 - kv0 + T - 1) / T);
  }
  plan.n_tiles = n_tiles;
  return placed;
}

int forward_packed_impl(ance_encoder_t e, const int32_t* ids_dev, const int32_t* lens_dev, const int32_t* lens_host, int B,
                        int L, float* out_dev, void* stream) {
  const ance_encoder_config& c = e->cfg;
  int dev = -1;
  ANCE_CUDA(cudaGetDevice(&dev));
  ANCE_REQUIRE(dev == e->device, "the encoder handle belongs to device %d but device %d is current", e->device, dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int cap_tiles = e->max_tokens / attn::kTile, max_seqs = e->max_tokens / 16;
  PackPlan plan;
  for (int first = 0; first < B;) {
    const int n = pack_chunk(lens_host, first, B, L, cap_tiles, max_seqs, e->varlen_align, plan);
    ANCE_REQUIRE(n > 0, "packed forward: sequence %d (%d tokens) does not fit a handle of max_tokens %d", first,
                 lens_host[first], e->max_tokens);
    // the plan arrays are read by the kernels of this chunk only; pageable cudaMemcpyAsync stages them before returning
    ANCE_CUDA(cudaMemcpyAsync(e->seq_row0, plan.row0.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
    ANCE_CUDA(cudaMemcpyAsync(e->row_lo, plan.lo.data(), plan.lo.size() * 4, cudaMemcpyHostToDevice, st));
    ANCE_CUDA(cudaMemcpyAsync(e->row_hi, plan.hi.data(), plan.hi.size() * 4, cudaMemcpyHostToDevice, st));
    ANCE_CUDA(cudaMemcpyAsync(e->tile_kv, plan.tile_kv.data(), plan.tile_kv.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
    const int32_t* ids = ids_dev + static_cast<size_t>(first) * L;
    float* out = out_dev + static_cast<size_t>(first) * c.hidden;
    const int rc = (e->fmt == tc05::kFmtBF16)
                       ? forward_impl<tc05::kFmtBF16>(e, ids, lens_dev + first, nullptr, n, L, out, st, plan.n_tiles)
                       : forward_impl<tc05::kFmtF16>(e, ids, lens_dev + first, nullptr, n, L, out, st, plan.n_tiles);
    if (rc) return rc;
    first += n;
  }
  return ANCE_OK;
}

}  // namespace

// host-only view of the tile packing (tests): plans the FIRST chunk of lens[0..B) for a handle of `max_tokens`
extern "C" int ance_dbg_pack_varlen(const int32_t* lens_host, int B, int max_tokens, int align, int32_t* row0_out,
                                    uint8_t* lo_out, uint8_t* hi_out, int* n_placed, int* n_tiles) {
  ANCE_REQUIRE(lens_host && row0_out && n_placed && n_tiles && B > 0 && max_tokens >= attn::kTile, "ance_dbg_pack_varlen: bad arguments");
  ANCE_REQUIRE(align == 1 || align == 16, "ance_dbg_pack_varlen: align must be 1 or 16");
  for (int b = 0; b < B; ++b) ANCE_REQUIRE(lens_host[b] >= 1 && lens_host[b] <= attn::kTile, "ance_dbg_pack_varlen: length %d out of range", lens_host[b]);
  PackPlan plan;
  *n_placed = pack_chunk(lens_host, 0, B, attn::kTile, max_tokens / attn::kTile, max_tokens / 16, align, plan);
  *n_tiles = plan.n_tiles;
  memcpy(row0_out, plan.row0.data(), plan.row0.size() * 4);
  for (size_t r = 0; r < plan.lo.size(); ++r) {   // tile-local
    const int t0 = static_cast<int>(r / attn::kTile) * attn::kTile;
    if (lo_out) lo_out[r] = static_cast<uint8_t>(plan.lo[r] - t0);
    if (hi_out) hi_out[r] = static_cast<uint8_t>(plan.hi[r] - t0);
  }
  return ANCE_OK;
}

extern "C" int ance_dbg_pack_packed(const int32_t* lens_host, int B, int L, int max_tokens, int align, int32_t* row0_out,
                                    int32_t* lo_out, int32_t* hi_out, int32_t* tile_kv_out, int* n_placed, int* n_tiles) {
  ANCE_REQUIRE(lens_host && row0_out && n_placed && n_tiles && B > 0, "ance_dbg_pack_packed: bad arguments");
  ANCE_REQUIRE(L > 0 && L <= 512 && max_tokens >= (L + attn::kTile - 1) / attn::kTile * attn::kTile,
               "ance_dbg_pack_packed: need 0 < L <= 512 and max_tokens >= L rounded up to 128 (L = %d, max_tokens = %d)", L, max_tokens);
  ANCE_REQUIRE(align == 1 || align == 16, "ance_dbg_pack_packed: align must be 1 or 16");
  for (int b = 0; b < B; ++b) ANCE_REQUIRE(lens_host[b] >= 1 && lens_host[b] <= L, "ance_dbg_pack_packed: length %d outside [1, %d]", lens_host[b], L);
  PackPlan plan;
  const int mt = max_tokens / attn::kTile * attn::kTile;
  *n_placed = pack_chunk(lens_host, 0, B, L, mt / attn::kTile, mt / 16, align, plan);
  *n_tiles = plan.n_tiles;
  memcpy(row0_out, plan.row0.data(), plan.row0.size() * 4);
  if (lo_out) memcpy(lo_out, plan.lo.data(), plan.lo.size() * 4);
  if (hi_out) memcpy(hi_out, plan.hi.data(), plan.hi.size() * 4);
  if (tile_kv_out) memcpy(tile_kv_out, plan.tile_kv.data(), plan.tile_kv.size() * sizeof(int2));
  return ANCE_OK;
}

extern "C" int ance_encoder_forward_varlen(ance_encoder_t e, const int32_t* ids_dev, const int32_t* lens_dev,
                                           const int32_t* lens_host, int B, int L, float* out_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_forward_varlen: null handle");
  ANCE_REQUIRE(ids_dev && lens_dev && lens_host && out_dev, "ance_encoder_forward_varlen: null buffer");
  ANCE_REQUIRE(B > 0 && L > 0 && L <= attn::kTile, "ance_encoder_forward_varlen: need B > 0 and 0 < L <= 128 (got B = %d, L = %d); "
               "longer sequences go through ance_encoder_forward", B, L);
  const ance_encoder_config& c = e->cfg;
  ANCE_REQUIRE(L + (c.arch == ANCE_ARCH_ROBERTA ? c.pad_id + 1 : 0) <= c.max_pos, "ance_encoder_forward_varlen: L = %d exceeds max_position_embeddings %d", L, c.max_pos);
  for (int b = 0; b < B; ++b)
    ANCE_REQUIRE(lens_host[b] >= 1 && lens_host[b] <= L, "ance_encoder_forward_varlen: length %d of sequence %d outside [1, %d]", lens_host[b], b, L);
  return forward_packed_impl(e, ids_dev, lens_dev, lens_host, B, L, out_dev, stream);
}

extern "C" int ance_encoder_forward_packed(ance_encoder_t e, const int32_t* ids_dev, const int32_t* lens_dev,
                                           const int32_t* lens_host, int B, int L, float* out_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_forward_packed: null handle");
  ANCE_REQUIRE(ids_dev && lens_dev && lens_host && out_dev, "ance_encoder_forward_packed: null buffer");
  ANCE_REQUIRE(B > 0 && L > 0 && L <= 512, "ance_encoder_forward_packed: need B > 0 and 0 < L <= 512 (got B = %d, L = %d)", B, L);
  const ance_encoder_config& c = e->cfg;
  ANCE_REQUIRE(L + (c.arch == ANCE_ARCH_ROBERTA ? c.pad_id + 1 : 0) <= c.max_pos, "ance_encoder_forward_packed: L = %d exceeds max_position_embeddings %d", L, c.max_pos);
  ANCE_REQUIRE(e->max_tokens >= (L + attn::kTile - 1) / attn::kTile * attn::kTile,
               "ance_encoder_forward_packed: L = %d needs a handle of max_tokens >= %d (got %d)", L,
               (L + attn::kTile - 1) / attn::kTile * attn::kTile, e->max_tokens);
  for (int b = 0; b < B; ++b)
    ANCE_REQUIRE(lens_host[b] >= 1 && lens_host[b] <= L, "ance_encoder_forward_packed: length %d of sequence %d outside [1, %d]", lens_host[b], b, L);
  return forward_packed_impl(e, ids_dev, lens_dev, lens_host, B, L, out_dev, stream);
}

extern "C" int ance_encoder_set_param(ance_encoder_t e, const char* name, double value) {
  ANCE_REQUIRE(e != nullptr && name != nullptr, "ance_encoder_set_param: null argument");
  if (!strcmp(name, "prune_last_layer")) e->prune_last_layer = value != 0;
  else if (!strcmp(name, "ln_rows_per_warp")) g_ln_rows_per_warp = static_cast<int>(value);
  else if (!strcmp(name, "varlen_align")) {
    ANCE_REQUIRE(value == 1 || value == 16, "varlen_align must be 1 or 16");
    e->varlen_align = static_cast<int>(value);
  }
  else { ance::set_error("ance_encoder_set_param: unknown parameter '%s'", name); return ANCE_ERR_INVALID; }
  return ANCE_OK;
}

extern "C" int ance_encoder_check(ance_encoder_t e, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_check: null handle");
  int err = 0;
  ANCE_CUDA(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
  ANCE_CUDA(cudaMemcpy(&err, e->err_flag, sizeof(int), cudaMemcpyDeviceToHost));
  if (err) {
    ANCE_CUDA(cudaMemset(e->err_flag, 0, sizeof(int)));
    if (err & 1) {
      ance::set_error("ance_encoder_forward: a token id outside [0, vocab_size) or a position past max_position_embeddings "
                      "was seen since the last check (the reference's embedding lookup raises an index error there)");
      return ANCE_ERR_INVALID;
    }
    ance::set_error("ance_encoder_forward: non-finite embeddings since the last check (%s)",
                    e->fmt == tc05::kFmtF16 ? "an activation left the fp16 range: create the encoder with operand_fmt = ANCE_FMT_BF16"
                                            : "NaN / inf in the weights or activations");
    return ANCE_ERR_UNSUPPORTED;
  }
  return ANCE_OK;
}

extern "C" int ance_encoder_debug_hidden(ance_encoder_t e, int layer, float* out_dev, void* stream) {
  ANCE_REQUIRE(e != nullptr, "ance_encoder_debug_hidden: null handle");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t H = e->cfg.hidden;
  if (layer < 0) {  // enable capture for batches up to 4096 tokens
    if (!e->dbg) {
      e->dbg_tokens = std::min(e->max_tokens, 4096);
      e->dbg = dev_alloc<uint16_t>(e, static_cast<size_t>(e->cfg.n_layer + 1) * e->dbg_tokens * H);
      ANCE_REQUIRE(e->dbg != nullptr, "ance_encoder_debug_hidden: allocation failed");
    }
    return ANCE_OK;
  }
  ANCE_REQUIRE(e->dbg != nullptr, "ance_encoder_debug_hidden: capture not enabled (call with layer = -1 first)");
  ANCE_REQUIRE(layer <= e->cfg.n_layer && out_dev, "ance_encoder_debug_hidden: bad layer or null buffer");
  const size_t n = static_cast<size_t>(e->dbg_tokens) * H;
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  if (e->fmt == tc05::kFmtBF16) act16_to_f32_kernel<tc05::kFmtBF16><<<blocks, 256, 0, st>>>(e->dbg + static_cast<size_t>(layer) * n, out_dev, n);
  else act16_to_f32_kernel<tc05::kFmtF16><<<blocks, 256, 0, st>>>(e->dbg + static_cast<size_t>(layer) * n, out_dev, n);
  ANCE_CUDA(cudaGetLastError());
  return ANCE_OK;
}

// ------------------------------------------------------------------------------------------------
// test hooks: the encoder's own GEMM, attention and LayerNorm launches on caller buffers
// ------------------------------------------------------------------------------------------------
namespace {

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

extern "C" int ance_dbg_linear(int fmt, const void* A_dev, int64_t lda, int M, const void* W_dev, int N, int K,
                               const float* bias_dev, const void* R_dev, int64_t ldr, int act, void* C16_dev,
                               float* C32_dev, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_linear: unknown operand format %d", fmt);
  ANCE_REQUIRE(A_dev && W_dev && (C16_dev || C32_dev), "ance_dbg_linear: null operand or no output");
  ANCE_REQUIRE(M > 0 && N > 0 && K > 0 && K % 8 == 0 && N % 8 == 0, "ance_dbg_linear: need M, N, K > 0 and N, K multiples of 8 (M=%d N=%d K=%d)", M, N, K);
  ANCE_REQUIRE(lda >= K && lda % 8 == 0, "ance_dbg_linear: lda = %lld must be >= K = %d and a multiple of 8", static_cast<long long>(lda), K);
  ANCE_REQUIRE(!R_dev || (ldr >= N && ldr % 8 == 0 && ldr <= INT32_MAX), "ance_dbg_linear: ldr = %lld must be >= N = %d and a multiple of 8", static_cast<long long>(ldr), N);
  ANCE_REQUIRE(act >= 0 && act <= 2, "ance_dbg_linear: act must be 0 (none), 1 (GELU, erfc form) or 2 (GELU, logistic form), got %d", act);
  ANCE_REQUIRE(aligned16(A_dev) && aligned16(W_dev) && aligned16(bias_dev) && aligned16(R_dev) && aligned16(C16_dev) && aligned16(C32_dev),
               "ance_dbg_linear: every buffer must be 16-byte aligned");
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* A = reinterpret_cast<const uint16_t*>(A_dev);
  const auto* W = reinterpret_cast<const uint16_t*>(W_dev);
  const auto* R = reinterpret_cast<const uint16_t*>(R_dev);
  auto* C = reinterpret_cast<uint16_t*>(C16_dev);
  const size_t ldr_ = R ? static_cast<size_t>(ldr) : 0;
  if (fmt == ANCE_FMT_BF16) return linear<tc05::kFmtBF16>(A, static_cast<size_t>(lda), M, W, N, K, bias_dev, R, act, C, C32_dev, st, ance::kClsGemm, ldr_);
  return linear<tc05::kFmtF16>(A, static_cast<size_t>(lda), M, W, N, K, bias_dev, R, act, C, C32_dev, st, ance::kClsGemm, ldr_);
}

extern "C" int ance_dbg_attention(int fmt, const void* qkv_dev, int n_tokens, int L, int heads, const float* kbias_dev,
                                  const int32_t* row_lo_dev, const int32_t* row_hi_dev, const int32_t* tile_kv_dev,
                                  void* ctx_dev, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_attention: unknown operand format %d", fmt);
  ANCE_REQUIRE(qkv_dev && ctx_dev && kbias_dev, "ance_dbg_attention: null buffer");
  ANCE_REQUIRE(aligned16(qkv_dev) && aligned16(ctx_dev), "ance_dbg_attention: qkv and ctx must be 16-byte aligned");
  ANCE_REQUIRE(heads >= 1 && heads <= 16, "ance_dbg_attention: heads = %d outside [1, 16]", heads);
  ANCE_REQUIRE(n_tokens > 0 && L > 0 && L <= 512, "ance_dbg_attention: need n_tokens > 0 and 0 < L <= 512 (n_tokens = %d, L = %d)", n_tokens, L);
  const bool varlen = row_lo_dev != nullptr;
  if (varlen) {
    ANCE_REQUIRE(row_hi_dev && n_tokens % attn::kTile == 0, "ance_dbg_attention: a row plan needs row_hi and n_tokens a multiple of 128");
    ANCE_REQUIRE((L > attn::kTile) == (tile_kv_dev != nullptr), "ance_dbg_attention: tile_kv is required for L > 128 and only then");
  } else {
    ANCE_REQUIRE(!row_hi_dev && !tile_kv_dev, "ance_dbg_attention: row_hi / tile_kv without row_lo");
    ANCE_REQUIRE((L % attn::kTile == 0) || (attn::kTile % L == 0 && L >= 8), "ance_dbg_attention: L = %d unsupported (need a multiple of 128 up to 512, or a divisor of 128)", L);
    ANCE_REQUIRE(n_tokens % L == 0, "ance_dbg_attention: n_tokens = %d is not a multiple of L = %d", n_tokens, L);
  }
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AttentionLaunch a;
  int rc = make_attention(a, reinterpret_cast<const uint16_t*>(qkv_dev), reinterpret_cast<uint16_t*>(ctx_dev), n_tokens, L,
                          heads, kbias_dev, row_lo_dev, row_hi_dev, reinterpret_cast<const int2*>(tile_kv_dev));
  if (rc) return rc;
  if (fmt == ANCE_FMT_BF16) {
    if ((rc = set_attention_attrs<tc05::kFmtBF16>())) return rc;
    return run_attention<tc05::kFmtBF16>(a, st);
  }
  if ((rc = set_attention_attrs<tc05::kFmtF16>())) return rc;
  return run_attention<tc05::kFmtF16>(a, st);
}

extern "C" int ance_dbg_layer_norm(int fmt, const void* in_dev, int in_f32, int64_t in_ld, int rows, int H,
                                   const float* gamma_dev, const float* beta_dev, float eps, void* out16_dev,
                                   float* out32_dev, int rows_per_warp, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_layer_norm: unknown operand format %d", fmt);
  ANCE_REQUIRE(in_dev && gamma_dev && beta_dev && (out16_dev || out32_dev), "ance_dbg_layer_norm: null buffer or no output");
  ANCE_REQUIRE(rows > 0 && H > 0 && H % 256 == 0 && H <= 1024, "ance_dbg_layer_norm: need rows > 0 and H in {256, 512, 768, 1024} (rows = %d, H = %d)", rows, H);
  ANCE_REQUIRE(in_ld >= H && in_ld % 8 == 0, "ance_dbg_layer_norm: in_ld = %lld must be >= H and a multiple of 8", static_cast<long long>(in_ld));
  ANCE_REQUIRE(rows_per_warp >= 1 && rows_per_warp <= 4, "ance_dbg_layer_norm: rows_per_warp must be 1, 2, 3 or 4, got %d", rows_per_warp);
  ANCE_REQUIRE(aligned16(in_dev) && aligned16(gamma_dev) && aligned16(beta_dev) && aligned16(out16_dev) && aligned16(out32_dev),
               "ance_dbg_layer_norm: every buffer must be 16-byte aligned");
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int saved = g_ln_rows_per_warp;
  g_ln_rows_per_warp = rows_per_warp;
  const int rc = (fmt == ANCE_FMT_BF16)
                     ? layer_norm<tc05::kFmtBF16>(in_dev, in_f32 != 0, static_cast<size_t>(in_ld), rows, H, gamma_dev, beta_dev, eps,
                                                  reinterpret_cast<uint16_t*>(out16_dev), out32_dev, st)
                     : layer_norm<tc05::kFmtF16>(in_dev, in_f32 != 0, static_cast<size_t>(in_ld), rows, H, gamma_dev, beta_dev, eps,
                                                 reinterpret_cast<uint16_t*>(out16_dev), out32_dev, st);
  g_ln_rows_per_warp = saved;
  return rc;
}

extern "C" int ance_dbg_attention_backward(int fmt, const void* qkv_dev, const float* kbias_dev, const void* dout_bf16_dev,
                                           int cls_only, int B, int L, int heads, float* dqkv_dev, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_attention_backward: unknown operand format %d", fmt);
  ANCE_REQUIRE(qkv_dev && kbias_dev && dout_bf16_dev && dqkv_dev, "ance_dbg_attention_backward: null buffer");
  ANCE_REQUIRE(heads >= 1 && heads <= 16, "ance_dbg_attention_backward: heads = %d outside [1, 16]", heads);
  ANCE_REQUIRE(B > 0 && L > 0 && L <= attn::kTile, "ance_dbg_attention_backward: need B > 0 and 0 < L <= 128 (B = %d, L = %d)", B, L);
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* qkv = reinterpret_cast<const uint16_t*>(qkv_dev);
  const auto* dout = reinterpret_cast<const uint16_t*>(dout_bf16_dev);
  if (fmt == ANCE_FMT_BF16) return attn_bwd<tc05::kFmtBF16>(qkv, kbias_dev, dout, cls_only != 0, dqkv_dev, B, L, heads, st);
  return attn_bwd<tc05::kFmtF16>(qkv, kbias_dev, dout, cls_only != 0, dqkv_dev, B, L, heads, st);
}

extern "C" int ance_dbg_layer_norm_backward(int fmt, const void* in_dev, int in_f32, int64_t in_ld, int rows, int H,
                                            const float* gamma_dev, float eps, const float* dy_dev, float* dx_dev,
                                            float* dgamma_dev, float* dbeta_dev, float* dsum_dev, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_layer_norm_backward: unknown operand format %d", fmt);
  ANCE_REQUIRE(in_dev && gamma_dev && dy_dev && dx_dev, "ance_dbg_layer_norm_backward: null buffer");
  ANCE_REQUIRE(rows > 0 && H > 0 && H % 256 == 0 && H <= 1024, "ance_dbg_layer_norm_backward: need rows > 0 and H in {256, 512, 768, 1024} (rows = %d, H = %d)", rows, H);
  ANCE_REQUIRE(in_ld >= H && in_ld % 8 == 0, "ance_dbg_layer_norm_backward: in_ld = %lld must be >= H and a multiple of 8", static_cast<long long>(in_ld));
  ANCE_REQUIRE(aligned16(in_dev) && aligned16(gamma_dev) && aligned16(dy_dev) && aligned16(dx_dev),
               "ance_dbg_layer_norm_backward: every buffer must be 16-byte aligned");
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* part = nullptr;
  ANCE_CUDA(cudaMallocAsync(&part, static_cast<size_t>(bwd::kLnBwdMaxBlocks) * 3 * H * 4, st));
  const int rc = (fmt == ANCE_FMT_BF16)
                     ? ln_bwd<tc05::kFmtBF16>(in_dev, in_f32 != 0, static_cast<size_t>(in_ld), rows, H, gamma_dev, eps, dy_dev, dx_dev, part, dgamma_dev, dbeta_dev, dsum_dev, st)
                     : ln_bwd<tc05::kFmtF16>(in_dev, in_f32 != 0, static_cast<size_t>(in_ld), rows, H, gamma_dev, eps, dy_dev, dx_dev, part, dgamma_dev, dbeta_dev, dsum_dev, st);
  ANCE_CUDA(cudaFreeAsync(part, st));
  return rc;
}

extern "C" int ance_dbg_gelu_backward(int fmt, const void* u_dev, float* g_dev, int64_t n, void* stream) {
  ANCE_REQUIRE(fmt == ANCE_FMT_FP16 || fmt == ANCE_FMT_BF16, "ance_dbg_gelu_backward: unknown operand format %d", fmt);
  ANCE_REQUIRE(u_dev && g_dev && n > 0, "ance_dbg_gelu_backward: null buffer or n <= 0");
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* u = reinterpret_cast<const uint16_t*>(u_dev);
  if (fmt == ANCE_FMT_BF16) bwd::gelu_bwd_kernel<tc05::kFmtBF16><<<ew_grid(n), 256, 0, st>>>(u, g_dev, static_cast<size_t>(n));
  else bwd::gelu_bwd_kernel<tc05::kFmtF16><<<ew_grid(n), 256, 0, st>>>(u, g_dev, static_cast<size_t>(n));
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}

extern "C" int ance_dbg_embedding_backward(const int32_t* ids_dev, int B, int L, int H, int roberta, int pad_id, int vocab,
                                           int max_pos, const float* word_dev, const float* pos_dev, const float* type_dev,
                                           const float* dE_dev, float* E_dev, float* dword_dev, float* dpos_dev,
                                           void* stream) {
  ANCE_REQUIRE(ids_dev && word_dev && pos_dev && type_dev && dE_dev && E_dev && dword_dev && dpos_dev,
               "ance_dbg_embedding_backward: null buffer");
  ANCE_REQUIRE(B > 0 && L > 0 && L <= attn::kTile && H > 0 && vocab > 0 && max_pos > 0,
               "ance_dbg_embedding_backward: need B, H, vocab, max_pos > 0 and 0 < L <= 128 (B = %d, L = %d)", B, L);
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int M = B * L;
  int32_t* pos_ids = nullptr;
  ANCE_CUDA(cudaMallocAsync(&pos_ids, static_cast<size_t>(M) * 4, st));
  bwd::embed_sum_kernel<<<B, 256, 0, st>>>(ids_dev, L, H, roberta != 0, pad_id, vocab, max_pos, word_dev, pos_dev, type_dev,
                                           E_dev, pos_ids);
  ANCE_CUDA(cudaMemsetAsync(dword_dev, 0, static_cast<size_t>(vocab) * H * 4, st));
  ANCE_CUDA(cudaMemsetAsync(dpos_dev, 0, static_cast<size_t>(max_pos) * H * 4, st));
  bwd::embed_scatter_kernel<<<M, 256, 0, st>>>(ids_dev, pos_ids, dE_dev, M, H, roberta != 0, pad_id, vocab, dword_dev, dpos_dev);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(2);
  ANCE_CUDA(cudaFreeAsync(pos_ids, st));
  return ANCE_OK;
}

extern "C" int ance_dbg_transpose_bf16(int src_kind, const void* src_dev, int64_t src_ld, int R, int C, void* dst_dev,
                                       int64_t dst_ld, void* stream) {
  ANCE_REQUIRE(src_kind >= 0 && src_kind <= 2, "ance_dbg_transpose_bf16: src_kind must be 0 (fp16), 1 (bf16) or 2 (fp32), got %d", src_kind);
  ANCE_REQUIRE(src_dev && dst_dev, "ance_dbg_transpose_bf16: null buffer");
  ANCE_REQUIRE(R > 0 && C > 0 && src_ld >= C && dst_ld >= R, "ance_dbg_transpose_bf16: need R, C > 0, src_ld >= C, dst_ld >= R");
  if (const int rc = require_sm90(nullptr)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t sl = static_cast<size_t>(src_ld), dl = static_cast<size_t>(dst_ld);
  auto* dst = reinterpret_cast<uint16_t*>(dst_dev);
  if (src_kind == 2) return transpose_bf16<2>(src_dev, sl, R, C, dst, dl, st);
  if (src_kind == 1) return transpose_bf16<1>(src_dev, sl, R, C, dst, dl, st);
  return transpose_bf16<0>(src_dev, sl, R, C, dst, dl, st);
}
