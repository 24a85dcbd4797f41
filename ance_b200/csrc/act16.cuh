// act16.cuh — the 16-bit storage format of encoder activations / weights as a compile-time trait.
//
// wgmma multiplies fp16 and bf16 operands at the same rate (fp32 accumulate either way); what differs is the
// rounding of everything that is STORED between kernels: bf16 keeps 8 significant bits (unit roundoff 2^-9), fp16 keeps
// 11 (2^-12).  The reference's forward is fp32 (model/models.py:149-157 under torch.no_grad, no autocast), so the encoder
// defaults to fp16 storage, which brings the embeddings 8x closer to the reference; bf16 stays
// selectable for checkpoints whose activations leave the fp16 range (|x| > 65504 -> inf -> NaN embeddings, which
// ance_encoder_check reports).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "tc05.cuh"

namespace act16 {

template <uint32_t FMT>
struct Act;

template <>
struct Act<tc05::kFmtBF16> {
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t v) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
  }
  static __device__ __forceinline__ float to_float(uint16_t v) { return __bfloat162float(__ushort_as_bfloat16(v)); }
  static __host__ uint16_t from_float_host(float f) {
    const __nv_bfloat16 h = __float2bfloat16_rn(f);
    uint16_t u;
    memcpy(&u, &h, 2);
    return u;
  }
};

template <>
struct Act<tc05::kFmtF16> {
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
  }
  static __device__ __forceinline__ float to_float(uint16_t v) { return __half2float(__ushort_as_half(v)); }
  static __host__ uint16_t from_float_host(float f) {
    const __half h = __float2half_rn(f);
    uint16_t u;
    memcpy(&u, &h, 2);
    return u;
  }
};

}  // namespace act16
