// common.h — error plumbing shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

#include "../../include/ance_b200.h"

namespace ance {

void set_error(const char* fmt, ...);  // defined in capi.cu
void count_launch(int n);

// device-time profile by kernel class (see ance_profile_enable in the header)
enum KernelClass { kClsGemm = 0, kClsAttn = 1, kClsNorm = 2, kClsQuant = 3, kClsCoarse = 4, kClsRescore = 5, kClsExact = 6,
                   kClsGemmQkv = 7, kClsGemmOut = 8, kClsGemmFfn1 = 9, kClsGemmFfn2 = 10, kClsOptim = 11,
                   kNumCls = 12 };
void prof_begin(int cls, cudaStream_t st);
void prof_end(int cls, cudaStream_t st);
struct ProfScope {
  int cls; cudaStream_t st;
  ProfScope(int c, cudaStream_t s) : cls(c), st(s) { prof_begin(cls, st); }
  ~ProfScope() { prof_end(cls, st); }
};

#define ANCE_CUDA(expr)                                                                       \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::ance::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ANCE_ERR_CUDA;                                                                   \
    }                                                                                         \
  } while (0)

#define ANCE_REQUIRE(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      ::ance::set_error(__VA_ARGS__);    \
      return ANCE_ERR_INVALID;           \
    }                                    \
  } while (0)

}  // namespace ance
