// encoder_bwd.cuh — kernels of the encoder's backward pass (sequences of up to 128 tokens), included by encoder.cu.
//
// The backward GEMMs (dgrad dX = dY W, wgrad dW = dY^T X) run on the forward's own wgmma mainloop and EpStore epilogue
// (encoder.cu: linear<kFmtBF16>) over transposed bf16 copies made here; everything else is in this file:
//   attn_bwd_kernel      softmax attention backward of one (sequence, head), S / P / dS held in shared memory
//   ln_bwd_kernel        LayerNorm backward of rows + per-block column partials of dgamma, dbeta and the bias gradient
//   colsum_*             deterministic two-stage column sums (bias gradients)
//   gelu_bwd_kernel      dU = dF * (Phi(u) + u phi(u)) from the saved 16-bit pre-activation
//   embed_sum_kernel / embed_scatter_kernel   embeddings: recompute the LayerNorm input, scatter-add the row gradients
//   transpose_bf16_kernel / f32_to_bf16_kernel / add_rows_kernel   operand plumbing
//   refresh_kernel       in-place weight refresh (ance_encoder_update_weights) in one launch
#pragma once
#include "act16.cuh"

namespace bwd {

constexpr int kLnBwdMaxBlocks = 264;   // column partials of ln_bwd_kernel: at most this many blocks (rows grid-strided)
constexpr int kColsumChunks = 128;     // row chunks of colsum_partial_kernel

__device__ __forceinline__ float bf16_to_float(uint16_t v) { return __bfloat162float(__ushort_as_bfloat16(v)); }
__device__ __forceinline__ uint16_t float_to_bf16(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }

// ------------------------------------------------------------------------------------------------
// Attention backward, one CTA per (sequence b, head h), L <= 128 keys.  With S = Q K^T / 8 + mask (natural units) and
// P = softmax(S) rebuilt from Q, K and the key bias exactly as the forward defines them (log2 domain, max subtracted):
//   dV = P^T dO ;  dP = dO V^T ;  dS = P o (dP - rowsum(P o dP)) ;  dQ = dS K / 8 ;  dK = dS^T Q / 8
// rowsum(P o dP) equals the usual rowsum(dO o O) in exact arithmetic; taken from the rebuilt P it needs no read of the
// forward's 16-bit O and makes every row of dS sum to zero up to fp32 rounding.
// Shared memory (fp32): Q, K, V, dO [L][65] (pitch 65: a warp reading 32 different rows at one column hits 32 banks) and
// P [L][L + 1], later overwritten by dS / 8.  All products are fp32 FMAs on the CUDA cores.
// dout: bf16 [B*L, H]; with cls_only only token 0 of each sequence has an upstream gradient and dout is [B, H] (the pruned
// last layer).  dqkv: fp32 [B*L, 3H] (Q | K | V, head-major inside each), every element of the sequence's rows written.
// ------------------------------------------------------------------------------------------------
constexpr int kAttnPitch = 65;
inline size_t attn_bwd_smem(int L) { return (static_cast<size_t>(4) * L * kAttnPitch + static_cast<size_t>(L) * (L + 1)) * 4; }

template <uint32_t FMT>
__global__ void __launch_bounds__(256) attn_bwd_kernel(const uint16_t* __restrict__ qkv, const float* __restrict__ kbias,
                                                       const uint16_t* __restrict__ dout, int cls_only,
                                                       float* __restrict__ dqkv, int L, int heads, float scale_log2) {
  using A16 = act16::Act<FMT>;
  extern __shared__ float sm[];
  const int b = blockIdx.x, h = blockIdx.y, H = heads * 64;
  const int PP = L + 1;
  float* sQ = sm;
  float* sK = sQ + L * kAttnPitch;
  float* sV = sK + L * kAttnPitch;
  float* sO = sV + L * kAttnPitch;   // dO
  float* sP = sO + L * kAttnPitch;
  const size_t tok0 = static_cast<size_t>(b) * L;
  for (int i = threadIdx.x; i < L * 64; i += blockDim.x) {
    const int r = i >> 6, d = i & 63;
    const uint16_t* row = qkv + (tok0 + r) * 3 * H + h * 64 + d;
    sQ[r * kAttnPitch + d] = A16::to_float(row[0]);
    sK[r * kAttnPitch + d] = A16::to_float(row[H]);
    sV[r * kAttnPitch + d] = A16::to_float(row[2 * H]);
    float go = 0.f;
    if (!cls_only) go = bf16_to_float(dout[(tok0 + r) * H + h * 64 + d]);
    else if (r == 0) go = bf16_to_float(dout[static_cast<size_t>(b) * H + h * 64 + d]);
    sO[r * kAttnPitch + d] = go;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // P: one warp per query row, lanes over keys
  for (int i = warp; i < L; i += 8) {
    float s[4];
    float m = -INFINITY;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int j = lane + 32 * t;
      s[t] = -INFINITY;
      if (j < L) {
        float acc = 0.f;
#pragma unroll 16
        for (int d = 0; d < 64; ++d) acc = fmaf(sQ[i * kAttnPitch + d], sK[j * kAttnPitch + d], acc);
        s[t] = fmaf(acc, scale_log2, kbias[tok0 + j]);
        m = fmaxf(m, s[t]);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      s[t] = (lane + 32 * t < L) ? exp2f(s[t] - m) : 0.f;
      sum += s[t];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (lane + 32 * t < L) sP[i * PP + lane + 32 * t] = s[t] * inv;
  }
  __syncthreads();
  // [L, 64] outputs: thread (r0, d) owns rows r0 + 4k, column d; within a warp r0 is uniform (the P / dS reads broadcast)
  const int d = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  float acc[32];
  // dV[j][d] = sum_i P[i][j] dO[i][d]
#pragma unroll
  for (int k = 0; k < 32; ++k) acc[k] = 0.f;
  for (int i = 0; i < L; ++i) {
    const float o = sO[i * kAttnPitch + d];
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (r0 + 4 * k < L) acc[k] = fmaf(sP[i * PP + r0 + 4 * k], o, acc[k]);
  }
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (r0 + 4 * k < L) dqkv[(tok0 + r0 + 4 * k) * 3 * H + 2 * H + h * 64 + d] = acc[k];
  __syncthreads();
  // dS / 8 over P: one warp per row
  for (int i = warp; i < L; i += 8) {
    float p[4], dp[4];
    float dsum = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int j = lane + 32 * t;
      p[t] = dp[t] = 0.f;
      if (j < L) {
        float a = 0.f;
#pragma unroll 16
        for (int c = 0; c < 64; ++c) a = fmaf(sO[i * kAttnPitch + c], sV[j * kAttnPitch + c], a);
        dp[t] = a;
        p[t] = sP[i * PP + j];
        dsum = fmaf(p[t], a, dsum);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (lane + 32 * t < L) sP[i * PP + lane + 32 * t] = p[t] * (dp[t] - dsum) * 0.125f;
  }
  __syncthreads();
  // dQ[i][d] = sum_j dS[i][j] K[j][d] / 8
#pragma unroll
  for (int k = 0; k < 32; ++k) acc[k] = 0.f;
  for (int j = 0; j < L; ++j) {
    const float kv = sK[j * kAttnPitch + d];
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (r0 + 4 * k < L) acc[k] = fmaf(sP[(r0 + 4 * k) * PP + j], kv, acc[k]);
  }
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (r0 + 4 * k < L) dqkv[(tok0 + r0 + 4 * k) * 3 * H + h * 64 + d] = acc[k];
  // dK[j][d] = sum_i dS[i][j] Q[i][d] / 8
#pragma unroll
  for (int k = 0; k < 32; ++k) acc[k] = 0.f;
  for (int i = 0; i < L; ++i) {
    const float q = sQ[i * kAttnPitch + d];
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (r0 + 4 * k < L) acc[k] = fmaf(sP[i * PP + r0 + 4 * k], q, acc[k]);
  }
#pragma unroll
  for (int k = 0; k < 32; ++k)
    if (r0 + 4 * k < L) dqkv[(tok0 + r0 + 4 * k) * 3 * H + H + h * 64 + d] = acc[k];
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward over rows, one warp per row (rows grid-strided over at most kLnBwdMaxBlocks blocks):
//   xhat = (x - mean) rstd, g = dy o gamma, dx = rstd (g - mean(g) - xhat mean(g o xhat))
// mean and rstd are recomputed from the saved LayerNorm input with the forward kernels' own arithmetic (same summation
// order, rsqrtf), so they are the forward's values bit for bit.  Every block also writes its column partials
//   part[blockIdx.x][0:H] = sum dy o xhat (dgamma), [H:2H] = sum dy (dbeta), [2H:3H] = sum dx (gradient of the bias of
// the linear layer whose output is x, or of the token-type row for the embedding LayerNorm), reduced over its 8 warps in
// a fixed order; colsum_final_kernel adds the blocks in a fixed order.  Deterministic.
// x: 16-bit (FMT) or fp32 at pitch x_ld; dy, dx: fp32 [rows, H].
// ------------------------------------------------------------------------------------------------
// out[c] = sum over the block's 8 warps (in warp order) of their per-lane column partials v
template <int NV>
__device__ __forceinline__ void block_colsum(float (&red)[8][NV * 256], const float (&v)[NV * 8], int warp, int lane, int H,
                                             float* __restrict__ out) {
#pragma unroll
  for (int j = 0; j < NV; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][(j * 32 + lane) * 8 + i] = v[j * 8 + i];
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][c];
    out[c] = t;
  }
  __syncthreads();
}

template <int NV, bool kInF32, uint32_t FMT>
__global__ void __launch_bounds__(256, 1) ln_bwd_kernel(const void* __restrict__ xin, size_t x_ld, int rows, int H,
                                                     const float* __restrict__ gamma, float eps,
                                                     const float* __restrict__ dy, float* __restrict__ dx,
                                                     float* __restrict__ part) {
  using A16 = act16::Act<FMT>;
  __shared__ float red[8][NV * 256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float cg[NV * 8], cb[NV * 8], cx[NV * 8];
#pragma unroll
  for (int i = 0; i < NV * 8; ++i) cg[i] = cb[i] = cx[i] = 0.f;
  for (int row = blockIdx.x * 8 + warp; row < rows; row += gridDim.x * 8) {
    float x[NV * 8], g[NV * 8];
    float sum = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (kInF32) {
        const float* r = reinterpret_cast<const float*>(xin) + static_cast<size_t>(row) * x_ld + col;
        const float4 a = __ldg(reinterpret_cast<const float4*>(r)), c = __ldg(reinterpret_cast<const float4*>(r + 4));
        x[v * 8 + 0] = a.x; x[v * 8 + 1] = a.y; x[v * 8 + 2] = a.z; x[v * 8 + 3] = a.w;
        x[v * 8 + 4] = c.x; x[v * 8 + 5] = c.y; x[v * 8 + 6] = c.z; x[v * 8 + 7] = c.w;
      } else {
        const uint16_t* r = reinterpret_cast<const uint16_t*>(xin) + static_cast<size_t>(row) * x_ld + col;
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
      const float dd = x[i] - mean;
      var = fmaf(dd, dd, var);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
    const float rstd = rsqrtf(var / H + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * 32 + lane) * 8;
      const float* dr = dy + static_cast<size_t>(row) * H + col;
      const float4 a = __ldg(reinterpret_cast<const float4*>(dr)), c = __ldg(reinterpret_cast<const float4*>(dr + 4));
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + col)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
      const float dv[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
      const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (x[v * 8 + i] - mean) * rstd;
        x[v * 8 + i] = xh;
        g[v * 8 + i] = dv[i] * gm[i];
        cg[v * 8 + i] = fmaf(dv[i], xh, cg[v * 8 + i]);
        cb[v * 8 + i] += dv[i];
        s1 += g[v * 8 + i];
        s2 = fmaf(g[v * 8 + i], xh, s2);
      }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, s);
      s2 += __shfl_xor_sync(0xffffffffu, s2, s);
    }
    const float m1 = s1 / H, m2 = s2 / H;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * 32 + lane) * 8;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[i] = rstd * (g[v * 8 + i] - m1 - x[v * 8 + i] * m2);
        cx[v * 8 + i] += o[i];
      }
      float* orow = dx + static_cast<size_t>(row) * H + col;
      *reinterpret_cast<float4*>(orow) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(orow + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
  }
  float* out = part + static_cast<size_t>(blockIdx.x) * 3 * H;
  block_colsum<NV>(red, cg, warp, lane, H, out);
  block_colsum<NV>(red, cb, warp, lane, H, out + H);
  block_colsum<NV>(red, cx, warp, lane, H, out + 2 * H);
}

// column partials of an fp32 [rows, N] matrix: part[chunk][c] = sum of rows chunk*per .. (chunk+1)*per, in row order
__global__ void colsum_partial_kernel(const float* __restrict__ a, int rows, int N, int per, float* __restrict__ part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  const int r0 = blockIdx.y * per, r1 = min(rows, r0 + per);
  float t = 0.f;
  for (int r = r0; r < r1; ++r) t += a[static_cast<size_t>(r) * N + c];
  part[static_cast<size_t>(blockIdx.y) * N + c] = t;
}

// out_s[c] = sum over blocks (in order) of part[blk][s * seg + c], for the up to three segments whose pointer is not null
__global__ void colsum_final_kernel(const float* __restrict__ part, int nblk, int N, int seg, float* o0, float* o1, float* o2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  float* o = c < seg ? o0 : c < 2 * seg ? o1 : o2;
  if (!o) return;
  float t = 0.f;
  for (int b = 0; b < nblk; ++b) t += part[static_cast<size_t>(b) * N + c];
  o[c % seg] = t;
}

// d/du gelu(u) = Phi(u) + u phi(u) (the exact erf GELU the forward's two closed forms approximate to <= 3.7e-6)
template <uint32_t FMT>
__global__ void gelu_bwd_kernel(const uint16_t* __restrict__ u16, float* __restrict__ g, size_t n) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float u = act16::Act<FMT>::to_float(u16[i]);
    const float d = 0.5f * erfcf(-u * 0.70710678118654752f) + u * 0.39894228040143268f * expf(-0.5f * u * u);
    g[i] *= d;
  }
}

// dst [C, dst_ld] bf16 = transpose of src [R, C] (row r at src + r * src_ld); columns R .. dst_ld of dst are zero-filled
// (the wgrad GEMM runs K = dst_ld).  kSrc: 0 fp16, 1 bf16, 2 fp32.  Block (32, 8), 32 x 32 tiles.
template <int kSrc>
__global__ void transpose_bf16_kernel(const void* __restrict__ src, size_t src_ld, int R, int C, uint16_t* __restrict__ dst,
                                      size_t dst_ld) {
  __shared__ float t[32][33];
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int r = r0 + k, c = c0 + threadIdx.x;
    float v = 0.f;
    if (r < R && c < C) {
      const size_t off = static_cast<size_t>(r) * src_ld + c;
      if (kSrc == 2) v = reinterpret_cast<const float*>(src)[off];
      else if (kSrc == 1) v = bf16_to_float(reinterpret_cast<const uint16_t*>(src)[off]);
      else v = __half2float(__ushort_as_half(reinterpret_cast<const uint16_t*>(src)[off]));
    }
    t[k][threadIdx.x] = v;
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int c = c0 + k, r = r0 + threadIdx.x;
    if (c < C && r < static_cast<int>(dst_ld)) dst[static_cast<size_t>(c) * dst_ld + r] = float_to_bf16(t[threadIdx.x][k]);
  }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ a, uint16_t* __restrict__ o, size_t n) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    o[i] = float_to_bf16(a[i]);
}

// In-place weight refresh: piece blockIdx.x of the table converts n fp32 values to the 16-bit format (to16) or copies them
constexpr uint32_t kRefreshChunk = 1u << 16;
struct RefreshPiece {
  const float* src;
  void* dst;
  uint32_t n, to16;
};

template <uint32_t FMT>
__global__ void __launch_bounds__(256) refresh_kernel(const RefreshPiece* __restrict__ table) {
  const RefreshPiece r = table[blockIdx.x];
  if (r.to16) {
    uint16_t* o = static_cast<uint16_t*>(r.dst);
    for (uint32_t i = threadIdx.x; i < r.n; i += blockDim.x) {
      if (FMT == tc05::kFmtBF16) o[i] = float_to_bf16(r.src[i]);
      else o[i] = __half_as_ushort(__float2half_rn(r.src[i]));
    }
  } else {
    float* o = static_cast<float*>(r.dst);
    for (uint32_t i = threadIdx.x; i < r.n; i += blockDim.x) o[i] = r.src[i];
  }
}

// dst[r * dst_row_stride] += src[r]   (rows of H fp32)
__global__ void add_rows_kernel(float* __restrict__ dst, size_t dst_row_stride, const float* __restrict__ src, int rows, int H) {
  const size_t n = static_cast<size_t>(rows) * H;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / H, c = i % H;
    dst[r * dst_row_stride * H + c] += src[i];
  }
}

// The embedding LayerNorm's input E = (word[id] + pos[p]) + type[0] (fp32, the forward's association) and the position id
// of every token of sequence b = blockIdx.x; positions follow the forward's rule (RoBERTa: cumsum of non-pad tokens + pad,
// pad tokens at pad; BERT: 0 .. L-1).  Ids / positions out of range are clamped as in the forward.
__global__ void __launch_bounds__(256) embed_sum_kernel(const int32_t* __restrict__ ids_all, int L, int H, int roberta,
                                                        int pad_id, int vocab, int max_pos, const float* __restrict__ word,
                                                        const float* __restrict__ pos, const float* __restrict__ type,
                                                        float* __restrict__ E, int32_t* __restrict__ pos_out) {
  __shared__ int s_pos[128];
  __shared__ int s_warp_cnt[8];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t* ids = ids_all + static_cast<size_t>(b) * L;
  {
    const int t = threadIdx.x;
    const int flag = (t < L && ids[t] != pad_id) ? 1 : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int pre = 0;
    for (int w2 = 0; w2 < warp; ++w2) pre += s_warp_cnt[w2];
    const int incl = pre + __popc(bal & ((2u << lane) - 1u));
    if (t < L) s_pos[t] = roberta ? (flag ? incl + pad_id : pad_id) : t;
    __syncthreads();
  }
  for (int t = warp; t < L; t += 8) {
    const size_t tok = static_cast<size_t>(b) * L + t;
    const int id = min(max(ids[t], 0), vocab - 1);
    const int ps = min(s_pos[t], max_pos - 1);
    if (lane == 0) pos_out[tok] = ps;
    for (int c = lane; c < H; c += 32)
      E[tok * H + c] = (word[static_cast<size_t>(id) * H + c] + pos[static_cast<size_t>(ps) * H + c]) + type[c];
  }
}

// word / position gradient rows += dE of every token (fp32 atomics: the order of the additions into a row that several
// tokens share is not deterministic).  The padding row of each table that the reference declares with padding_idx gets
// no gradient: word row pad_id always, position row pad_id for RoBERTa.
__global__ void embed_scatter_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ pos_ids,
                                     const float* __restrict__ dE, int M, int H, int roberta, int pad_id, int vocab,
                                     float* __restrict__ dword, float* __restrict__ dpos) {
  const int tok = blockIdx.x;
  if (tok >= M) return;
  const int raw = ids[tok];
  const int id = min(max(raw, 0), vocab - 1), ps = pos_ids[tok];
  const bool w_ok = raw != pad_id, p_ok = !(roberta && ps == pad_id);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const float g = dE[static_cast<size_t>(tok) * H + c];
    if (w_ok) atomicAdd(dword + static_cast<size_t>(id) * H + c, g);
    if (p_ok) atomicAdd(dpos + static_cast<size_t>(ps) * H + c, g);
  }
}

}  // namespace bwd
