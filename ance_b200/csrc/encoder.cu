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

// n_tiles > 0: variable-length packing — the plan (e->seq_row0 / row_lo / row_hi / tile_kv) is already on the device, the
// token matrix has n_tiles * 128 rows and the CLS rows are gathered by index.  With L > 128 sequences may span tiles.
template <uint32_t FMT>
int forward_impl(ance_encoder* e, const int32_t* ids_dev, const int32_t* lens_dev, const uint8_t* mask_dev, int B, int L,
                 float* out_dev, cudaStream_t st, int n_tiles = 0) {
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
  ep.ids = ids_dev; ep.lens = lens_dev; ep.mask = mask_dev;
  ep.B = B; ep.L = L; ep.H = H;
  ep.roberta = (c.arch == ANCE_ARCH_ROBERTA);
  ep.pad_id = c.pad_id; ep.vocab = c.vocab; ep.max_pos = c.max_pos;
  ep.word = e->word; ep.pos = e->pos; ep.type = e->type;
  ep.gamma = e->eg; ep.beta = e->eb; ep.eps = c.ln_eps;
  ep.X = e->X; ep.kbias = e->kbias; ep.err_flag = e->err_flag;
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
    if ((rc = linear<FMT>(e->X, H, M, d.wqkv, 3 * H, H, d.bqkv, nullptr, 0, e->QKV, nullptr, st, ance::kClsGemmQkv))) return rc;
    if ((rc = run_attention<FMT>(attn_launch, st))) return rc;
    // In the last layer only token 0 of every sequence is read downstream (models.py:49,193): run the
    // out-projection, FFN and both LayerNorms on those B rows only (strided TMA views, compact outputs).
    const bool cls_only = (e->prune_last_layer || varlen) && (l == c.n_layer - 1);
    const int Mr = cls_only ? B : M;                                    // rows processed from here on
    const uint16_t *ctx_a = e->CTX, *res_x = e->X;
    size_t pitch = cls_only ? static_cast<size_t>(L) * H : H;           // row pitch of CTX / X views
    if (cls_only && varlen) {   // the CLS rows sit at seq_row0[b]: gather them into compact [B, H] operands
      ance::ProfScope ps(ance::kClsNorm, st);
      gather_rows16_by_index_kernel<<<B, 96, 0, st>>>(e->CTX, e->seq_row0, B, H, e->cls_ctx);
      gather_rows16_by_index_kernel<<<B, 96, 0, st>>>(e->X, e->seq_row0, B, H, e->cls_x);
      ANCE_CUDA(cudaGetLastError());
      ance::count_launch(2);
      ctx_a = e->cls_ctx; res_x = e->cls_x; pitch = H;
    }
    if ((rc = linear<FMT>(ctx_a, pitch, Mr, d.wo, H, H, d.bo, res_x, 0, e->T, nullptr, st, ance::kClsGemmOut, pitch))) return rc;
    if ((rc = layer_norm<FMT>(e->T, false, H, Mr, H, d.ln1g, d.ln1b, c.ln_eps, e->X1, nullptr, st))) return rc;
    if ((rc = linear<FMT>(e->X1, H, Mr, d.w1, F, H, d.b1, nullptr, gelu_form(), e->FF, nullptr, st, ance::kClsGemmFfn1))) return rc;
    if ((rc = linear<FMT>(e->FF, F, Mr, d.w2, H, F, d.b2, e->X1, 0, e->T, nullptr, st, ance::kClsGemmFfn2))) return rc;
    if ((rc = layer_norm<FMT>(e->T, false, H, Mr, H, d.ln2g, d.ln2b, c.ln_eps, e->X, nullptr, st))) return rc;
    if (e->dbg && M <= e->dbg_tokens)  // with cls_only the first B rows hold the CLS rows of the last layer
      ANCE_CUDA(cudaMemcpyAsync(e->dbg + static_cast<size_t>(l + 1) * e->dbg_tokens * H, e->X, static_cast<size_t>(Mr) * H * 2, cudaMemcpyDeviceToDevice, st));
  }
  const size_t cls_pitch = (e->prune_last_layer || varlen) ? static_cast<size_t>(H) : static_cast<size_t>(L) * H;
  // K7: CLS rows (token 0 of every sequence) -> head
  if (c.has_head) {
    // A = the CLS rows of X ([B, H] compact after the pruned last layer, else row pitch L*H)
    if ((rc = linear<FMT>(e->X, cls_pitch, B, e->head_w, H, H, e->head_b, nullptr, 0, nullptr, e->head_tmp, st))) return rc;
    if ((rc = layer_norm<FMT>(e->head_tmp, true, H, B, H, e->head_g, e->head_bt, 1e-5f, nullptr, out_dev, st))) return rc;
  } else {
    ance::ProfScope ps(ance::kClsNorm, st);
    gather_rows_f32_kernel<FMT><<<B, 256, 0, st>>>(e->X, cls_pitch, B, H, out_dev);
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
