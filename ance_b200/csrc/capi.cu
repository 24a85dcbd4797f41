// capi.cu — error state, version, launch counter and the bring-up GEMM hook of libance_b200.so.
#include <atomic>
#include <mutex>
#include <string.h>
#include <vector>

#include "common.h"
#include "gemm_store.cuh"

namespace ance {

static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---- profile ----
static bool g_prof_on = false;
static std::mutex g_prof_mu;
static std::vector<cudaEvent_t> g_ev_pool;
struct Span { cudaEvent_t a, b; };
static std::vector<Span> g_spans[kNumCls];
static cudaEvent_t g_open[kNumCls];
static double g_ms[kNumCls];
static int64_t g_cnt[kNumCls];

static cudaEvent_t get_event() {
  if (!g_ev_pool.empty()) { cudaEvent_t e = g_ev_pool.back(); g_ev_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
void prof_begin(int cls, cudaStream_t st) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_open[cls] = get_event();
  cudaEventRecord(g_open[cls], st);
}
void prof_end(int cls, cudaStream_t st) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEvent_t b = get_event();
  cudaEventRecord(b, st);
  g_spans[cls].push_back({g_open[cls], b});
}

}  // namespace ance

extern "C" const char* ance_version(void) { return "ance_b200 0.1 (sm_90a)"; }
extern "C" const char* ance_last_error(void) { return ance::g_err; }
extern "C" int64_t ance_launch_count(void) { return ance::g_launches.load(); }

extern "C" int ance_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(ance::g_prof_mu);
  ance::g_prof_on = on != 0;
  return ANCE_OK;
}

extern "C" int ance_profile_read(double* ms_by_class, int64_t* launches_by_class, int n, int reset) {
  ANCE_REQUIRE(ms_by_class && launches_by_class && n > 0 && n <= ance::kNumCls, "ance_profile_read: bad arguments");
  ANCE_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(ance::g_prof_mu);
  for (int c = 0; c < ance::kNumCls; ++c) {
    for (auto& s : ance::g_spans[c]) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, s.a, s.b) == cudaSuccess) { ance::g_ms[c] += ms; ance::g_cnt[c] += 1; }
      ance::g_ev_pool.push_back(s.a);
      ance::g_ev_pool.push_back(s.b);
    }
    ance::g_spans[c].clear();
  }
  for (int c = 0; c < n; ++c) { ms_by_class[c] = ance::g_ms[c]; launches_by_class[c] = ance::g_cnt[c]; }
  if (reset) for (int c = 0; c < ance::kNumCls; ++c) { ance::g_ms[c] = 0; ance::g_cnt[c] = 0; }
  return ANCE_OK;
}

namespace {

template <int BN, int STAGES, int CG, uint32_t FMT>
int run_dbg(const void* A, const void* B, int M, int N, int K, const float* bias, const void* R, int act, void* C,
            float* C32, cudaStream_t st) {
  constexpr int EW = 4;
  using Ep = gemm::EpStore<BN, EW>;
  CUtensorMap tmA, tmB;
  if (!tc05_host::make_tmap_2d_16b(&tmA, A, M, K, K, gemm::BM) ||
      !tc05_host::make_tmap_2d_16b(&tmB, B, N, K, K, BN / CG)) {
    ance::set_error("cuTensorMapEncodeTiled failed (M=%d N=%d K=%d)", M, N, K);
    return ANCE_ERR_CUDA;
  }
  gemm::WorkShape ws = gemm::make_shape(M, N, K, BN, CG, 0);
  typename Ep::Params p;
  memset(&p, 0, sizeof(p));
  if (C && !gemm::make_store_tmap(&p.tmC, C, M, N, N)) {
    ance::set_error("cuTensorMapEncodeTiled failed for the output (M=%d N=%d)", M, N);
    return ANCE_ERR_CUDA;
  }
  if (C && R && !gemm::make_store_tmap(&p.tmR, const_cast<void*>(R), M, N, N)) {
    ance::set_error("cuTensorMapEncodeTiled failed for the residual (M=%d N=%d)", M, N);
    return ANCE_ERR_CUDA;
  }
  p.C = reinterpret_cast<uint16_t*>(C);
  p.C32 = C32;
  p.bias = bias;
  p.R = reinterpret_cast<const uint16_t*>(R);
  p.ldc = N;
  p.ldc32 = N;
  p.ldr = N;
  p.act = act;
  ANCE_CUDA((gemm::launch<Ep, BN, STAGES, CG, EW, FMT>(tmA, tmB, ws, p, 0, st)));
  ance::count_launch(1);
  return ANCE_OK;
}

// 128 x 256 tiles on two MMA warpgroups (tc05_gemm_wide_kernel): 16-bit output only
template <uint32_t FMT>
int run_dbg_wide(const void* A, const void* B, int M, int N, int K, const float* bias, const void* R, int act, void* C,
                 float* C32, cudaStream_t st) {
  using Ep = gemm::EpStoreWide<>;
  ANCE_REQUIRE(C && !C32, "ance_dbg_gemm: variant 5 writes a 16-bit output only");
  CUtensorMap tmA, tmB;
  if (!tc05_host::make_tmap_2d_16b(&tmA, A, M, K, K, gemm::BM) ||
      !tc05_host::make_tmap_2d_16b(&tmB, B, N, K, K, gemm::kWideBN)) {
    ance::set_error("cuTensorMapEncodeTiled failed (M=%d N=%d K=%d)", M, N, K);
    return ANCE_ERR_CUDA;
  }
  gemm::WorkShape ws = gemm::make_shape(M, N, K, gemm::kWideBN, 1, 0);
  typename Ep::Params p;
  memset(&p, 0, sizeof(p));
  if (!gemm::make_store_wide_tmap(&p.tmC, C, M, N, N) ||
      (R && !gemm::make_store_wide_tmap(&p.tmR, const_cast<void*>(R), M, N, N))) {
    ance::set_error("cuTensorMapEncodeTiled failed for the output or residual (M=%d N=%d)", M, N);
    return ANCE_ERR_CUDA;
  }
  p.bias = bias;
  p.R = reinterpret_cast<const uint16_t*>(R);
  p.act = act;
  ANCE_CUDA((gemm::launch_wide<Ep, FMT>(tmA, tmB, ws, p, 0, st)));
  ance::count_launch(1);
  return ANCE_OK;
}

template <uint32_t FMT>
int dispatch_dbg(int variant, const void* A, const void* B, int M, int N, int K, const float* bias, const void* R,
                 int act, void* C, float* C32, cudaStream_t st) {
  switch (variant) {
    case 0: return run_dbg<128, 4, 1, FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    case 1: return run_dbg<128, 3, 1, FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    case 2: return run_dbg<128, 4, 2, FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    case 3: return run_dbg<64, 6, 2, FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    case 4: return run_dbg<64, 6, 1, FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    case 5: return run_dbg_wide<FMT>(A, B, M, N, K, bias, R, act, C, C32, st);
    default: ance::set_error("ance_dbg_gemm: unknown variant %d", variant); return ANCE_ERR_INVALID;
  }
}

}  // namespace

extern "C" int ance_dbg_gemm(const void* A_dev, const void* B_dev, int M, int N, int K, int fmt, int variant,
                             const float* bias_dev, const void* residual_bf16_dev, int act, void* C_bf16_dev,
                             float* C_f32_dev, void* stream) {
  ANCE_REQUIRE(A_dev && B_dev && M > 0 && N > 0 && K > 0, "ance_dbg_gemm: null operand or empty shape");
  ANCE_REQUIRE(K % 8 == 0 && N % 8 == 0, "ance_dbg_gemm: K and N must be multiples of 8 (16-byte rows)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (fmt == ANCE_FMT_BF16)
    return dispatch_dbg<tc05::kFmtBF16>(variant, A_dev, B_dev, M, N, K, bias_dev, residual_bf16_dev, act, C_bf16_dev,
                                        C_f32_dev, st);
  if (fmt == ANCE_FMT_FP16)
    return dispatch_dbg<tc05::kFmtF16>(variant, A_dev, B_dev, M, N, K, bias_dev, residual_bf16_dev, act, C_bf16_dev,
                                       C_f32_dev, st);
  ance::set_error("ance_dbg_gemm: unknown operand format %d", fmt);
  return ANCE_ERR_INVALID;
}
