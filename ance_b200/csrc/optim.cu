// optim.cu — the LAMB (ance_lamb_step) and AdamW (ance_adamw_step) optimizer steps as multi-tensor updates: three
// launches (LAMB) or one (AdamW) per call whatever the number of tensors, no host synchronisation, no float atomics.
//
// LAMB:
//   moments : per (tensor, chunk) block, m <- b1 m + (1 - b1) g, v <- b2 v + (1 - b2) g^2, u = m / (sqrt v + eps) + wd p
//             in registers; the block's sums of p^2 and u^2 (fp64) go to its slot of a per-block scratch.
//   norms   : per tensor, the fixed-order sum of its blocks' slots -> w = min(||p||, 10), a = ||u||, r = w / a (1 when
//             either is 0), written to norms[3 t .. 3 t + 2].
//   update  : per (tensor, chunk) block, u recomputed from m, v and p exactly as the first pass formed it, then
//             p <- p - lr (adam ? 1 : r) u.
// Traffic: the first pass reads p, g, m, v and writes m, v; the second reads p, m, v and writes p: 40 bytes per element.
//
// AdamW (transformers 2.3.0's AdamW.step): per (tensor, chunk) block, the same moment update (rounded as torch's addcmul
// rounds it, see adamw_update), then
//   p <- p + (-step_size) (m / (sqrt v + eps)),  then, only when decay = lr weight_decay > 0, p <- p + (-decay) p
// with step_size (bias correction already applied) and decay per tensor: reads p, g, m, v and writes p, m, v, 28 bytes
// per element, no norms and no second pass.
//
// Either table travels as a __grid_constant__ kernel parameter (< 32 KB, CUDA >= 12.1), rebuilt per call, so nothing
// on the host can be overwritten while an earlier step is still in flight.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "common.h"

namespace {

constexpr int kMaxTensors = 512;   // table capacity of either step (kernel-parameter space)
constexpr int kMaxHyper = 16;      // distinct (lr, betas, eps, weight decay) tuples per call; for AdamW (betas, eps)
constexpr int kThreads = 256;
constexpr int kChunk = 16384;      // elements per block (a multiple of 4 * kThreads * kIlp)
constexpr int kIlp = 4;            // float4 loads in flight per thread and array
constexpr uint8_t kScalar = 0xff;  // head[t]: the four arrays do not share an alignment; every element goes scalar

struct Hyper {
  float b1, c1, b2, c2, eps, wd, neg_lr, pad;   // c1 = 1 - b1 and c2 = 1 - b2 rounded once from double
};

struct Table {
  float* p[kMaxTensors];
  const float* g[kMaxTensors];
  float* m[kMaxTensors];
  float* v[kMaxTensors];
  int64_t n[kMaxTensors];
  int32_t blk0[kMaxTensors + 1];   // first block of each tensor; blk0[n_tensors] = the grid
  uint8_t hyp[kMaxTensors];        // index into h
  uint8_t head[kMaxTensors];       // scalar elements before the first 16-byte aligned one, or kScalar
  Hyper h[kMaxHyper];
  double2* part;                   // [grid] (sum p^2, sum u^2) of each block
  float* norms;                    // [n_tensors, 3] (w, a, r)
  int n_tensors;
  int adam;
};
static_assert(sizeof(Table) <= 32764, "the tensor table must fit the kernel-parameter space");

// AdamW's table: the same tensor list, the (betas, eps) tuples in h (wd and neg_lr unused, 0), and per tensor the two scalars that
// differ with each parameter's step count and group.
struct AdamWTable {
  float* p[kMaxTensors];
  const float* g[kMaxTensors];
  float* m[kMaxTensors];
  float* v[kMaxTensors];
  int64_t n[kMaxTensors];
  int32_t blk0[kMaxTensors + 1];
  uint8_t hyp[kMaxTensors];
  uint8_t head[kMaxTensors];
  Hyper h[kMaxHyper];
  float neg_step[kMaxTensors];    // -step_size, rounded once from double
  float neg_decay[kMaxTensors];   // -lr weight_decay rounded once from double; 0 when lr weight_decay <= 0 (no decay)
  int n_tensors;
};
static_assert(sizeof(AdamWTable) <= 32764, "the tensor table must fit the kernel-parameter space");

template <class Tab>
__device__ __forceinline__ int find_tensor(const Tab& T, int b) {
  int lo = 0, hi = T.n_tensors;   // blk0[lo] <= b < blk0[hi]; empty tensors (blk0[t] == blk0[t + 1]) are skipped
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (T.blk0[mid] <= b) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float adam_step(float p, float m, float v, const Hyper& H) {
  float u = __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), H.eps));
  if (H.wd != 0.f) u = __fmaf_rn(H.wd, p, u);
  return u;
}

// m and v updated in place; returns u.  The operation order and roundings are those of the eager fp32 step.
__device__ __forceinline__ float moments(float p, float g, float& m, float& v, const Hyper& H) {
  m = __fmaf_rn(H.c1, g, __fmul_rn(m, H.b1));
  v = __fmaf_rn(__fmul_rn(H.c2, g), g, __fmul_rn(v, H.b2));
  return adam_step(p, m, v, H);
}

// The elements block b owns: vectors [v0, v1) of the aligned body and, for the tensor's first block, the scalar head and
// tail; or scalar elements [s0, s1) when the tensor cannot be vectorised.
struct Span {
  int t;
  int64_t v0, v1, s0, s1, tail0;
  int head;
};

template <class Tab>
__device__ __forceinline__ Span span_of(const Tab& T, int b) {
  Span s;
  s.t = find_tensor(T, b);
  const int64_t c = b - T.blk0[s.t], n = T.n[s.t];
  const int head = T.head[s.t];
  if (head == kScalar) {
    s.head = 0;
    s.v0 = s.v1 = 0;
    s.s0 = c * kChunk;
    s.s1 = min(n, s.s0 + kChunk);
    s.tail0 = n;
  } else {
    const int64_t nv = (n - head) >> 2;
    s.head = c == 0 ? head : 0;
    s.v0 = c * (kChunk / 4);
    s.v1 = min(nv, s.v0 + kChunk / 4);
    s.s0 = s.s1 = 0;
    s.tail0 = c == 0 ? head + 4 * nv : n;   // the tail [tail0, n) is the first block's
  }
  return s;
}

__device__ __forceinline__ void block_sum_store(double sp, double su, double2* out) {
  __shared__ double2 red[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sp += __shfl_xor_sync(0xffffffffu, sp, o);
    su += __shfl_xor_sync(0xffffffffu, su, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = make_double2(sp, su);
  __syncthreads();
  if (threadIdx.x == 0) {
    double2 a = red[0];
#pragma unroll
    for (int i = 1; i < kThreads / 32; ++i) { a.x += red[i].x; a.y += red[i].y; }
    *out = a;
  }
}

__global__ void __launch_bounds__(kThreads) lamb_moments_kernel(const __grid_constant__ Table T) {
  const Span s = span_of(T, blockIdx.x);
  const Hyper H = T.h[T.hyp[s.t]];
  float* __restrict__ p = T.p[s.t];
  const float* __restrict__ g = T.g[s.t];
  float* __restrict__ m = T.m[s.t];
  float* __restrict__ v = T.v[s.t];
  const int64_t n = T.n[s.t];
  double sp = 0.0, su = 0.0;

  auto scalar = [&](int64_t i) {
    const float pi = p[i];
    float mi = m[i], vi = v[i];
    const float u = moments(pi, g[i], mi, vi, H);
    m[i] = mi;
    v[i] = vi;
    sp = fma((double)pi, (double)pi, sp);
    su = fma((double)u, (double)u, su);
  };
  for (int64_t i = threadIdx.x; i < s.head; i += kThreads) scalar(i);
  for (int64_t i = s.s0 + threadIdx.x; i < s.s1; i += kThreads) scalar(i);
  for (int64_t i = s.tail0 + threadIdx.x; i < n; i += kThreads) scalar(i);

  const int hd = T.head[s.t] == kScalar ? 0 : T.head[s.t];
  const float4* __restrict__ p4 = reinterpret_cast<const float4*>(p + hd);
  const float4* __restrict__ g4 = reinterpret_cast<const float4*>(g + hd);
  float4* __restrict__ m4 = reinterpret_cast<float4*>(m + hd);
  float4* __restrict__ v4 = reinterpret_cast<float4*>(v + hd);
  for (int64_t base = s.v0 + threadIdx.x; base < s.v1; base += kIlp * kThreads) {
    float4 P[kIlp], G[kIlp], M[kIlp], V[kIlp];
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) { P[k] = p4[i]; G[k] = g4[i]; M[k] = m4[i]; V[k] = v4[i]; }
    }
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) {
        const float u0 = moments(P[k].x, G[k].x, M[k].x, V[k].x, H);
        const float u1 = moments(P[k].y, G[k].y, M[k].y, V[k].y, H);
        const float u2 = moments(P[k].z, G[k].z, M[k].z, V[k].z, H);
        const float u3 = moments(P[k].w, G[k].w, M[k].w, V[k].w, H);
        m4[i] = M[k];
        v4[i] = V[k];
        sp = fma((double)P[k].x, (double)P[k].x, sp);
        sp = fma((double)P[k].y, (double)P[k].y, sp);
        sp = fma((double)P[k].z, (double)P[k].z, sp);
        sp = fma((double)P[k].w, (double)P[k].w, sp);
        su = fma((double)u0, (double)u0, su);
        su = fma((double)u1, (double)u1, su);
        su = fma((double)u2, (double)u2, su);
        su = fma((double)u3, (double)u3, su);
      }
    }
  }
  block_sum_store(sp, su, T.part + blockIdx.x);
}

__global__ void __launch_bounds__(kThreads) lamb_norms_kernel(const __grid_constant__ Table T) {
  const int t = blockIdx.x;
  double sp = 0.0, su = 0.0;
  for (int b = T.blk0[t] + threadIdx.x; b < T.blk0[t + 1]; b += kThreads) {
    const double2 x = T.part[b];
    sp += x.x;
    su += x.y;
  }
  __shared__ double2 tot;
  block_sum_store(sp, su, &tot);
  __syncthreads();
  if (threadIdx.x == 0) {
    const float norm_p = (float)sqrt(tot.x);
    const float w = norm_p > 10.f ? 10.f : norm_p;   // clamp(0, 10); NaN stays NaN
    const float a = (float)sqrt(tot.y);
    const float r = (w == 0.f || a == 0.f) ? 1.f : __fdiv_rn(w, a);
    T.norms[3 * t + 0] = w;
    T.norms[3 * t + 1] = a;
    T.norms[3 * t + 2] = r;
  }
}

__global__ void __launch_bounds__(kThreads) lamb_update_kernel(const __grid_constant__ Table T) {
  const Span s = span_of(T, blockIdx.x);
  const Hyper H = T.h[T.hyp[s.t]];
  float* __restrict__ p = T.p[s.t];
  const float* __restrict__ m = T.m[s.t];
  const float* __restrict__ v = T.v[s.t];
  const int64_t n = T.n[s.t];
  const float alpha = T.adam ? H.neg_lr : __fmul_rn(H.neg_lr, T.norms[3 * s.t + 2]);

  auto scalar = [&](int64_t i) {
    const float pi = p[i];
    p[i] = __fmaf_rn(alpha, adam_step(pi, m[i], v[i], H), pi);
  };
  for (int64_t i = threadIdx.x; i < s.head; i += kThreads) scalar(i);
  for (int64_t i = s.s0 + threadIdx.x; i < s.s1; i += kThreads) scalar(i);
  for (int64_t i = s.tail0 + threadIdx.x; i < n; i += kThreads) scalar(i);

  const int hd = T.head[s.t] == kScalar ? 0 : T.head[s.t];
  float4* __restrict__ p4 = reinterpret_cast<float4*>(p + hd);
  const float4* __restrict__ m4 = reinterpret_cast<const float4*>(m + hd);
  const float4* __restrict__ v4 = reinterpret_cast<const float4*>(v + hd);
  for (int64_t base = s.v0 + threadIdx.x; base < s.v1; base += kIlp * kThreads) {
    float4 P[kIlp], M[kIlp], V[kIlp];
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) { P[k] = p4[i]; M[k] = m4[i]; V[k] = v4[i]; }
    }
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) {
        float4 o;
        o.x = __fmaf_rn(alpha, adam_step(P[k].x, M[k].x, V[k].x, H), P[k].x);
        o.y = __fmaf_rn(alpha, adam_step(P[k].y, M[k].y, V[k].y, H), P[k].y);
        o.z = __fmaf_rn(alpha, adam_step(P[k].z, M[k].z, V[k].z, H), P[k].z);
        o.w = __fmaf_rn(alpha, adam_step(P[k].w, M[k].w, V[k].w, H), P[k].w);
        p4[i] = o;
      }
    }
  }
}

// p after one AdamW step; m and v updated in place.  The roundings are those of the eager fp32 step on the GPU (each
// checked bit for bit against torch's CUDA kernels, tests/test_gpu_adamw.py):
//   m = fma(1 - b1, g, m b1)        exp_avg.mul_(b1).add_(g, alpha=1 - b1): the product rounded, then add's a + alpha b
//                                   contracted into one FMA (as LAMB's moments())
//   v = fma(1 - b2, g g, v b2)      exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2): addcmul's a + alpha (b c), the square
//                                   rounded first.  LAMB's moments() forms fma((1 - b2) g, g, v b2) instead, which differs
//                                   from torch in the last bit of a few elements per million; it is left as it is.
//   q = m / (sqrt(v) + eps)         exp_avg_sq.sqrt().add_(eps), then addcdiv's b / c: square root, sum and quotient each
//                                   rounded to nearest (IEEE, no fast math)
//   p = fma(-step_size, q, p)       addcdiv_'s a + alpha (b / c), contracted into one FMA
//   p = fma(-decay, p, p)           p.add_(p, alpha=-lr wd) on the already-updated p, one FMA; skipped when neg_decay is 0
// The scalars are rounded to fp32 once from double on the host, as torch rounds a Python scalar to the op's fp32 type.
__device__ __forceinline__ float adamw_update(float p, float g, float& m, float& v, const Hyper& H, float neg_step,
                                              float neg_decay) {
  m = __fmaf_rn(H.c1, g, __fmul_rn(m, H.b1));
  v = __fmaf_rn(H.c2, __fmul_rn(g, g), __fmul_rn(v, H.b2));
  p = __fmaf_rn(neg_step, __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), H.eps)), p);
  return neg_decay != 0.f ? __fmaf_rn(neg_decay, p, p) : p;
}

__global__ void __launch_bounds__(kThreads) adamw_step_kernel(const __grid_constant__ AdamWTable T) {
  const Span s = span_of(T, blockIdx.x);
  const Hyper H = T.h[T.hyp[s.t]];
  const float ns = T.neg_step[s.t], nd = T.neg_decay[s.t];
  float* __restrict__ p = T.p[s.t];
  const float* __restrict__ g = T.g[s.t];
  float* __restrict__ m = T.m[s.t];
  float* __restrict__ v = T.v[s.t];
  const int64_t n = T.n[s.t];

  auto scalar = [&](int64_t i) {
    float mi = m[i], vi = v[i];
    p[i] = adamw_update(p[i], g[i], mi, vi, H, ns, nd);
    m[i] = mi;
    v[i] = vi;
  };
  for (int64_t i = threadIdx.x; i < s.head; i += kThreads) scalar(i);
  for (int64_t i = s.s0 + threadIdx.x; i < s.s1; i += kThreads) scalar(i);
  for (int64_t i = s.tail0 + threadIdx.x; i < n; i += kThreads) scalar(i);

  const int hd = T.head[s.t] == kScalar ? 0 : T.head[s.t];
  float4* __restrict__ p4 = reinterpret_cast<float4*>(p + hd);
  const float4* __restrict__ g4 = reinterpret_cast<const float4*>(g + hd);
  float4* __restrict__ m4 = reinterpret_cast<float4*>(m + hd);
  float4* __restrict__ v4 = reinterpret_cast<float4*>(v + hd);
  for (int64_t base = s.v0 + threadIdx.x; base < s.v1; base += kIlp * kThreads) {
    float4 P[kIlp], G[kIlp], M[kIlp], V[kIlp];
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) { P[k] = p4[i]; G[k] = g4[i]; M[k] = m4[i]; V[k] = v4[i]; }
    }
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
      const int64_t i = base + k * kThreads;
      if (i < s.v1) {
        P[k].x = adamw_update(P[k].x, G[k].x, M[k].x, V[k].x, H, ns, nd);
        P[k].y = adamw_update(P[k].y, G[k].y, M[k].y, V[k].y, H, ns, nd);
        P[k].z = adamw_update(P[k].z, G[k].z, M[k].z, V[k].z, H, ns, nd);
        P[k].w = adamw_update(P[k].w, G[k].w, M[k].w, V[k].w, H, ns, nd);
        p4[i] = P[k];
        m4[i] = M[k];
        v4[i] = V[k];
      }
    }
  }
}

inline unsigned misalign(const void* q) { return (unsigned)(reinterpret_cast<uintptr_t>(q) & 15u); }

// Checks tensor t's arguments and enters its pointers, size, scalar head and first block into T; `blocks` (the blocks of
// the tensors before t) advances past t's.  fn names the entry point in error messages.
template <class Tab>
int add_tensor(Tab& T, int t, const char* fn, float* p, const float* g, float* m, float* v, int64_t ne,
               int64_t& blocks) {
  ANCE_REQUIRE(ne >= 0, "%s: tensor %d has numel %lld < 0", fn, t, (long long)ne);
  const void* ptrs[4] = {p, g, m, v};
  for (int k = 0; k < 4; ++k) {
    ANCE_REQUIRE(ne == 0 || ptrs[k], "%s: tensor %d (numel %lld) has a null pointer", fn, t, (long long)ne);
    ANCE_REQUIRE((reinterpret_cast<uintptr_t>(ptrs[k]) & 3u) == 0,
                 "%s: tensor %d has a pointer that is not 4-byte aligned", fn, t);
  }
  T.p[t] = p;
  T.g[t] = g;
  T.m[t] = m;
  T.v[t] = v;
  T.n[t] = ne;
  const unsigned a = misalign(p);
  int64_t chunks;
  if (misalign(g) == a && misalign(m) == a && misalign(v) == a) {
    const int64_t head = ne < (int64_t)((16 - a) % 16 / 4) ? ne : (int64_t)((16 - a) % 16 / 4);
    T.head[t] = (uint8_t)head;
    const int64_t nv = (ne - head) / 4;
    chunks = ne == 0 ? 0 : (nv == 0 ? 1 : (nv + kChunk / 4 - 1) / (kChunk / 4));
  } else {
    T.head[t] = kScalar;
    chunks = (ne + kChunk - 1) / kChunk;
  }
  T.blk0[t] = (int32_t)blocks;
  blocks += chunks;
  if (blocks > INT32_MAX) {
    ance::set_error("%s: more than 2^31 blocks of %d elements in one call", fn, kChunk);
    return ANCE_ERR_UNSUPPORTED;
  }
  return ANCE_OK;
}

// The index of H in T.h, entered when new; -1 when the call already holds kMaxHyper other tuples (the caller sets the
// error).
template <class Tab>
int hyper_slot(Tab& T, int& n_hyper, const Hyper& H) {
  int k = 0;
  while (k < n_hyper && memcmp(&T.h[k], &H, sizeof(H)) != 0) ++k;
  if (k == n_hyper) {
    if (n_hyper == kMaxHyper) return -1;
    T.h[n_hyper++] = H;
  }
  return k;
}

}  // namespace

extern "C" int ance_lamb_step(int n, float* const* p_dev, const float* const* g_dev, float* const* m_dev,
                              float* const* v_dev, const int64_t* numel, const double* hyper, int adam,
                              float* norms_dev, void* stream) {
  ANCE_REQUIRE(n >= 0, "ance_lamb_step: n = %d < 0", n);
  if (n == 0) return ANCE_OK;
  ANCE_REQUIRE(p_dev && g_dev && m_dev && v_dev && numel && hyper && norms_dev,
               "ance_lamb_step: null table array or norms output");
  if (n > kMaxTensors) {
    ance::set_error("ance_lamb_step: %d tensors in one call; the table holds at most %d (split the call)", n,
                    kMaxTensors);
    return ANCE_ERR_UNSUPPORTED;
  }
  ANCE_REQUIRE((reinterpret_cast<uintptr_t>(norms_dev) & 3u) == 0, "ance_lamb_step: norms output not 4-byte aligned");
  static thread_local Table T;   // 24 KB: kept off the stack; copied into the launches' parameter buffers
  memset(&T, 0, sizeof(T));
  int n_hyper = 0;
  int64_t blocks = 0;
  for (int t = 0; t < n; ++t) {
    const int rc = add_tensor(T, t, "ance_lamb_step", p_dev[t], g_dev[t], m_dev[t], v_dev[t], numel[t], blocks);
    if (rc != ANCE_OK) return rc;
    const double* hp = hyper + 5 * t;   // lr, beta1, beta2, eps, weight_decay
    const Hyper H = {(float)hp[1], (float)(1.0 - hp[1]), (float)hp[2], (float)(1.0 - hp[2]), (float)hp[3],
                     (float)hp[4], (float)(-hp[0]), 0.f};
    const int k = hyper_slot(T, n_hyper, H);
    if (k < 0) {
      ance::set_error("ance_lamb_step: more than %d distinct (lr, betas, eps, weight_decay) in one call", kMaxHyper);
      return ANCE_ERR_UNSUPPORTED;
    }
    T.hyp[t] = (uint8_t)k;
  }
  T.blk0[n] = (int32_t)blocks;
  T.n_tensors = n;
  T.adam = adam ? 1 : 0;
  T.norms = norms_dev;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ance::ProfScope prof(ance::kClsOptim, st);
  if (blocks > 0) ANCE_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&T.part), blocks * sizeof(double2), st));
  if (blocks > 0) lamb_moments_kernel<<<(unsigned)blocks, kThreads, 0, st>>>(T);
  lamb_norms_kernel<<<n, kThreads, 0, st>>>(T);
  if (blocks > 0) lamb_update_kernel<<<(unsigned)blocks, kThreads, 0, st>>>(T);
  const cudaError_t launched = cudaGetLastError();
  if (blocks > 0) ANCE_CUDA(cudaFreeAsync(T.part, st));
  ANCE_CUDA(launched);
  ance::count_launch(blocks > 0 ? 3 : 1);
  return ANCE_OK;
}

extern "C" int ance_adamw_step(int n, float* const* p_dev, const float* const* g_dev, float* const* m_dev,
                               float* const* v_dev, const int64_t* numel, const double* hyper, void* stream) {
  ANCE_REQUIRE(n >= 0, "ance_adamw_step: n = %d < 0", n);
  if (n == 0) return ANCE_OK;
  ANCE_REQUIRE(p_dev && g_dev && m_dev && v_dev && numel && hyper, "ance_adamw_step: null table array");
  if (n > kMaxTensors) {
    ance::set_error("ance_adamw_step: %d tensors in one call; the table holds at most %d (split the call)", n,
                    kMaxTensors);
    return ANCE_ERR_UNSUPPORTED;
  }
  static thread_local AdamWTable T;   // 28 KB: kept off the stack; copied into the launch's parameter buffer
  memset(&T, 0, sizeof(T));
  int n_hyper = 0;
  int64_t blocks = 0;
  for (int t = 0; t < n; ++t) {
    const int rc = add_tensor(T, t, "ance_adamw_step", p_dev[t], g_dev[t], m_dev[t], v_dev[t], numel[t], blocks);
    if (rc != ANCE_OK) return rc;
    const double* hp = hyper + 5 * t;   // step_size, beta1, beta2, eps, decay = lr weight_decay
    const Hyper H = {(float)hp[1], (float)(1.0 - hp[1]), (float)hp[2], (float)(1.0 - hp[2]), (float)hp[3], 0.f, 0.f,
                     0.f};
    const int k = hyper_slot(T, n_hyper, H);
    if (k < 0) {
      ance::set_error("ance_adamw_step: more than %d distinct (betas, eps) in one call", kMaxHyper);
      return ANCE_ERR_UNSUPPORTED;
    }
    T.hyp[t] = (uint8_t)k;
    T.neg_step[t] = (float)(-hp[0]);
    T.neg_decay[t] = hp[4] > 0.0 ? (float)(-hp[4]) : 0.f;
  }
  T.blk0[n] = (int32_t)blocks;
  T.n_tensors = n;

  if (blocks == 0) return ANCE_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ance::ProfScope prof(ance::kClsOptim, st);
  adamw_step_kernel<<<(unsigned)blocks, kThreads, 0, st>>>(T);
  ANCE_CUDA(cudaGetLastError());
  ance::count_launch(1);
  return ANCE_OK;
}
