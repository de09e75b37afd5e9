// Library GEMMs for the in/out projections (the boundary of the custom-kernel span).
//
// An alternative to this library's own projection kernels (proj_gemm.cuh): plain library GEMMs (cuBLASLt), selected
// with HYENA_B200_PROJ=lt or when the user opted into TF32.  What this file adds over torch.bmm is the choice of
// cuBLASLt build: PyTorch 2.11+cu128 bundles cuBLAS 12.8, whose fp32 GEMM is the CUDA-core SGEMM.  The CUDA 12.9
// toolkit ships cuBLASLt 12.9, which has CUBLAS_COMPUTE_32F_EMULATED_16BFX9: fp32 GEMM emulated on the bf16
// tensor cores with nine bf16 products per fp32 product -- fp32-level accuracy (no TF32 rounding), a
// multiple of the SGEMM rate.  That library is dlopen()ed by absolute path into a private handle
// (RTLD_LOCAL), so PyTorch's own cuBLAS is untouched.  If it cannot be loaded the entry point reports
// failure and the Python side keeps using torch.bmm (also a GPU library GEMM; no CPU path anywhere).
#include <cublasLt.h>
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

#include "../../include/hyena_b200.h"
#include "launch.h"

namespace hy {
int api_fail(const char* fmt, ...);   // api.cu

struct LtApi {
  void* so = nullptr;
  cublasLtHandle_t handles[64] = {nullptr};      // one per device, created on first use there
  size_t version = 0;
  decltype(&cublasLtCreate) Create;
  decltype(&cublasLtGetVersion) GetVersion;
  decltype(&cublasLtMatmul) Matmul;
  decltype(&cublasLtMatmulDescCreate) DescCreate;
  decltype(&cublasLtMatmulDescDestroy) DescDestroy;
  decltype(&cublasLtMatmulDescSetAttribute) DescSet;
  decltype(&cublasLtMatrixLayoutCreate) LayoutCreate;
  decltype(&cublasLtMatrixLayoutDestroy) LayoutDestroy;
  decltype(&cublasLtMatrixLayoutSetAttribute) LayoutSet;
  decltype(&cublasLtMatmulPreferenceCreate) PrefCreate;
  decltype(&cublasLtMatmulPreferenceDestroy) PrefDestroy;
  decltype(&cublasLtMatmulPreferenceSetAttribute) PrefSet;
  decltype(&cublasLtMatmulAlgoGetHeuristic) Heuristic;
};

static LtApi g_lt;
static std::mutex g_lt_mu;
static int g_lt_state = 0;     // 0 untried, 1 ok, -1 unavailable
static char g_lt_why[256] = "";

static const char* kCandidates[] = {
    "/usr/local/cuda/lib64/libcublasLt.so.12.9.1.4", "/usr/local/cuda-12.9/lib64/libcublasLt.so.12",
    "/usr/local/cuda/lib64/libcublasLt.so.12", nullptr};

static bool lt_load() {
  std::lock_guard<std::mutex> lk(g_lt_mu);
  if (g_lt_state) return g_lt_state > 0;
  g_lt_state = -1;
  const char* env = getenv("HYENA_B200_CUBLASLT");
  void* so = nullptr;
  if (env && *env) so = dlopen(env, RTLD_NOW | RTLD_LOCAL);
  for (int i = 0; !so && kCandidates[i]; ++i) so = dlopen(kCandidates[i], RTLD_NOW | RTLD_LOCAL);
  if (!so) { snprintf(g_lt_why, sizeof(g_lt_why), "cuBLASLt 12.9 not found: %s", dlerror()); return false; }
#define HY_SYM(field, name)                                                              \
  g_lt.field = reinterpret_cast<decltype(g_lt.field)>(dlsym(so, name));                  \
  if (!g_lt.field) { snprintf(g_lt_why, sizeof(g_lt_why), "missing symbol %s", name); return false; }
  HY_SYM(Create, "cublasLtCreate") HY_SYM(GetVersion, "cublasLtGetVersion") HY_SYM(Matmul, "cublasLtMatmul")
  HY_SYM(DescCreate, "cublasLtMatmulDescCreate") HY_SYM(DescDestroy, "cublasLtMatmulDescDestroy")
  HY_SYM(DescSet, "cublasLtMatmulDescSetAttribute") HY_SYM(LayoutCreate, "cublasLtMatrixLayoutCreate")
  HY_SYM(LayoutDestroy, "cublasLtMatrixLayoutDestroy") HY_SYM(LayoutSet, "cublasLtMatrixLayoutSetAttribute")
  HY_SYM(PrefCreate, "cublasLtMatmulPreferenceCreate") HY_SYM(PrefDestroy, "cublasLtMatmulPreferenceDestroy")
  HY_SYM(PrefSet, "cublasLtMatmulPreferenceSetAttribute") HY_SYM(Heuristic, "cublasLtMatmulAlgoGetHeuristic")
#undef HY_SYM
  g_lt.version = g_lt.GetVersion();
  if (g_lt.version < 120900) {
    snprintf(g_lt_why, sizeof(g_lt_why), "cuBLASLt %zu has no BF16x9 fp32 emulation (need >= 12.9)", g_lt.version);
    return false;
  }
  g_lt.so = so;
  g_lt_state = 1;
  return true;
}

struct Plan {
  cublasLtMatmulDesc_t desc = nullptr;
  cublasLtMatrixLayout_t a = nullptr, b = nullptr, c = nullptr;
  cublasLtMatmulAlgo_t algo;
  size_t ws = 0;
  bool ok = false;
};
// first element: device ordinal (heuristics / algos are per device)
using Key = std::tuple<int, int, int, int, int, int, int, int, int, int, long long, long long, long long, int, int>;
static std::map<Key, Plan> g_plans;

static void plan_destroy(Plan& p) {
  if (p.a) g_lt.LayoutDestroy(p.a);
  if (p.b) g_lt.LayoutDestroy(p.b);
  if (p.c) g_lt.LayoutDestroy(p.c);
  if (p.desc) g_lt.DescDestroy(p.desc);
  p = Plan();
}

}  // namespace hy

using namespace hy;

extern "C" {

/* 1 if the BF16x9-emulating cuBLASLt could be loaded, else 0 (reason via hyena_b200_last_error). */
HY_API int hyena_b200_gemm_available(void) {
  if (lt_load()) return 1;
  api_fail("%s", g_lt_why);
  return 0;
}

/* Column-major strided-batched C = alpha * op(A) op(B) + beta * C (+ bias[m] broadcast over columns),
 * fp32 in / fp32 out; emulate: 1 = CUBLAS_COMPUTE_32F_EMULATED_16BFX9, 2 = CUBLAS_COMPUTE_32F_FAST_TF32 (only when
 * the caller opted into TF32), 0 = plain CUBLAS_COMPUTE_32F.  op = 'N' (0) or 'T' (1).  workspace: >= 32 MiB recommended. */
HY_API int hyena_b200_gemm(int transa, int transb, int m, int n, int k, float alpha, const float* A, int lda,
                           long long strideA, const float* B, int ldb, long long strideB, float beta, float* C,
                           int ldc, long long strideC, int batch, const float* bias, int emulate, void* workspace,
                           size_t workspace_bytes, void* stream) {
  if (!lt_load()) return api_fail("%s", g_lt_why);
  if (m < 1 || n < 1 || k < 1 || batch < 1 || !A || !B || !C) return api_fail("gemm: bad arguments");
  std::lock_guard<std::mutex> lk(g_lt_mu);
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return api_fail("gemm: unsupported device ordinal %d", dev);
  if (!g_lt.handles[dev] && g_lt.Create(&g_lt.handles[dev]) != CUBLAS_STATUS_SUCCESS) {
    g_lt.handles[dev] = nullptr;
    return api_fail("cublasLtCreate failed on device %d", dev);
  }
  cublasLtHandle_t handle = g_lt.handles[dev];
  Key key{dev, transa, transb, m, n, k, lda, ldb, ldc, batch, strideA, strideB, strideC, bias != nullptr, emulate};
  Plan& p = g_plans[key];
  if (!p.ok) {
    plan_destroy(p);                       // a previous attempt may have left partial objects behind
    // emulate: 0 = plain fp32, 1 = BF16x9 emulation (fp32-level accuracy), 2 = TF32 (opt-in: torch allow_tf32)
    const cublasComputeType_t ct = emulate == 1 ? CUBLAS_COMPUTE_32F_EMULATED_16BFX9
                                   : emulate == 2 ? CUBLAS_COMPUTE_32F_FAST_TF32 : CUBLAS_COMPUTE_32F;
    if (g_lt.DescCreate(&p.desc, ct, CUDA_R_32F) != CUBLAS_STATUS_SUCCESS) {
      g_plans.erase(key);
      return api_fail("cublasLtMatmulDescCreate failed");
    }
    cublasOperation_t ta = transa ? CUBLAS_OP_T : CUBLAS_OP_N, tb = transb ? CUBLAS_OP_T : CUBLAS_OP_N;
    g_lt.DescSet(p.desc, CUBLASLT_MATMUL_DESC_TRANSA, &ta, sizeof(ta));
    g_lt.DescSet(p.desc, CUBLASLT_MATMUL_DESC_TRANSB, &tb, sizeof(tb));
    if (bias) {
      cublasLtEpilogue_t ep = CUBLASLT_EPILOGUE_BIAS;
      g_lt.DescSet(p.desc, CUBLASLT_MATMUL_DESC_EPILOGUE, &ep, sizeof(ep));
    }
    auto mk = [&](cublasLtMatrixLayout_t* l, int rows, int cols, int ld, long long stride) {
      if (g_lt.LayoutCreate(l, CUDA_R_32F, rows, cols, ld) != CUBLAS_STATUS_SUCCESS) return false;
      int32_t bc = batch;
      int64_t st = stride;
      g_lt.LayoutSet(*l, CUBLASLT_MATRIX_LAYOUT_BATCH_COUNT, &bc, sizeof(bc));
      g_lt.LayoutSet(*l, CUBLASLT_MATRIX_LAYOUT_STRIDED_BATCH_OFFSET, &st, sizeof(st));
      return true;
    };
    if (!mk(&p.a, transa ? k : m, transa ? m : k, lda, strideA) || !mk(&p.b, transb ? n : k, transb ? k : n, ldb, strideB) ||
        !mk(&p.c, m, n, ldc, strideC)) {
      plan_destroy(p);
      g_plans.erase(key);
      return api_fail("cublasLtMatrixLayoutCreate failed");
    }
    cublasLtMatmulPreference_t pref = nullptr;
    g_lt.PrefCreate(&pref);
    size_t wsb = workspace ? workspace_bytes : 0;
    g_lt.PrefSet(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &wsb, sizeof(wsb));
    if (bias) {   // heuristics need a (dummy) bias pointer attribute to be present
      const void* bp = bias;
      g_lt.DescSet(p.desc, CUBLASLT_MATMUL_DESC_BIAS_POINTER, &bp, sizeof(bp));
    }
    cublasLtMatmulHeuristicResult_t res;
    int found = 0;
    cublasStatus_t st = g_lt.Heuristic(handle, p.desc, p.a, p.b, p.c, p.c, pref, 1, &res, &found);
    g_lt.PrefDestroy(pref);
    if (st != CUBLAS_STATUS_SUCCESS || found < 1) {
      plan_destroy(p);
      g_plans.erase(key);
      return api_fail("cublasLt heuristic found no algorithm (status %d) for m=%d n=%d k=%d emulate=%d", (int)st, m, n, k, emulate);
    }
    p.algo = res.algo;
    p.ws = res.workspaceSize;
    p.ok = true;
  }
  if (bias) {
    const void* bp = bias;
    g_lt.DescSet(p.desc, CUBLASLT_MATMUL_DESC_BIAS_POINTER, &bp, sizeof(bp));
  }
  if (p.ws > workspace_bytes) return api_fail("gemm workspace too small (%zu needed)", p.ws);
  cublasStatus_t st = g_lt.Matmul(handle, p.desc, &alpha, A, p.a, B, p.b, &beta, C, p.c, C, p.c, &p.algo, workspace,
                                  p.ws, (cudaStream_t)stream);
  if (st != CUBLAS_STATUS_SUCCESS) return api_fail("cublasLtMatmul failed with status %d", (int)st);
  return 0;
}

}  // extern "C"
