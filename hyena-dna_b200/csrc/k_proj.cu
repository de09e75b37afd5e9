// Launchers of the wgmma projection GEMMs (proj_gemm.cuh).
#include <cstdint>
#include <cstring>

#include "../../include/hyena_b200.h"
#include "launch.h"
#include "proj_gemm.cuh"

namespace hy {

static_assert(FN_GELU_TANH == HYENA_B200_GELU_TANH && FN_GELU_ERF == HYENA_B200_GELU_ERF, "activation codes of the C ABI");

size_t proj_wimg_bytes(int N, int K) {
  const int NT = 128;
  return pg::wimg_floats(N, K, NT) * sizeof(float);
}

// cuTensorMapEncodeTiled through the runtime's driver entry point lookup (no libcuda link dependency)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// fp32 matrix (rows x cols, row pitch = cols) -> tensor map with box (box_cols x box_rows)
static bool make_tmap(CUtensorMap* m, const float* base, unsigned long long rows, unsigned long long cols, unsigned box_cols,
                      unsigned box_rows, bool swizzle128) {
  EncodeTiledFn f = encode_tiled();
  if (!f) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(float)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return f(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 tensor (d2, d1, d0) with d0 contiguous -> 3-D tensor map with box (b0 x b1 x 1)
static bool make_tmap3(CUtensorMap* m, const float* base, unsigned long long d0, unsigned long long d1, unsigned long long d2,
                       unsigned b0, unsigned b1) {
  EncodeTiledFn f = encode_tiled();
  if (!f) return false;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * sizeof(float), d0 * d1 * sizeof(float)};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return f(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int NT, int ACT, int OUT, int FN = FN_NONE>
static cudaError_t go(pg::Args a, int sms, cudaStream_t s, int kind = K_PROJ_GEMM) {
  auto kern = pg::proj_gemm_kernel<NT, ACT, OUT, FN>;
  CUtensorMap tmap;
  memset(&tmap, 0, sizeof(tmap));
  if (a.vec) {
    const bool ok = (ACT == pg::ACT_ROW)
        ? make_tmap(&tmap, a.act, (unsigned long long)a.B * a.L, (unsigned long long)a.K, 32, 128, true)
        : make_tmap(&tmap, a.act, (unsigned long long)a.B * a.K, (unsigned long long)a.L, 132, 32, false);
    if (!ok) a.vec = 0;                    // no driver entry point / unencodable shape: lanes stage the tiles instead
  }
  const size_t smem = pg::Cfg<NT>::SMEM + (a.fir ? (size_t)a.K * 12 : 0);
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long ntiles = (long long)a.B * a.mtiles_per_b * a.ntiles_n;
  const int grid = (int)(ntiles < sms ? ntiles : sms);
  prof_begin(kind, s);
  kern<<<grid, pg::kThreads, smem, s>>>(a, tmap);
  prof_end(kind, s);
  return cudaGetLastError();
}

template <int NT>
static cudaError_t by_layout(const pg::Args& a, int act_layout, int out_layout, int sms, cudaStream_t s) {
  if (act_layout == pg::ACT_ROW && out_layout == pg::OUT_CH) return go<NT, pg::ACT_ROW, pg::OUT_CH>(a, sms, s);
  if (act_layout == pg::ACT_ROW && out_layout == pg::OUT_ROW) return go<NT, pg::ACT_ROW, pg::OUT_ROW>(a, sms, s);
  if (act_layout == pg::ACT_CH && out_layout == pg::OUT_CH) return go<NT, pg::ACT_CH, pg::OUT_CH>(a, sms, s);
  if (act_layout == pg::ACT_CH && out_layout == pg::OUT_ROW) return go<NT, pg::ACT_CH, pg::OUT_ROW>(a, sms, s);
  return cudaErrorInvalidValue;
}

cudaError_t launch_proj_gemm(const float* act, int act_layout, const float* W, int ldw, int w_transposed, const float* bias,
                             const float* fir, float* out, int out_layout, int B, int L, int K, int N, int l0, int ln,
                             float* wimg, cudaStream_t s, int fn, const float* aux) {
  const int NT = 128;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t total = pg::wimg_floats(N, K, NT);
  int pblocks = (int)((total + 255) / 256);
  if (pblocks > 4 * sms) pblocks = 4 * sms;
  prof_begin(K_PROJ_PREP, s);
  pg::proj_prep_kernel<<<pblocks, 256, 0, s>>>(W, ldw, w_transposed, N, K, NT, wimg);
  prof_end(K_PROJ_PREP, s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  pg::Args a;
  a.act = act; a.wimg = wimg; a.out = out; a.bias = bias; a.fir = fir; a.aux = aux;
  a.B = B; a.L = L; a.K = K; a.N = N; a.l0 = l0; a.ln = ln;
  // TMA needs 16-byte aligned rows (global stride a multiple of 16 bytes) and, for the channel-major box, a 16-byte
  // aligned first position
  if (act_layout == pg::ACT_ROW) a.vec = (K % 4 == 0);
  else a.vec = (L % 4 == 0) && (l0 % 4 == 0);
  a.kchunks = (K + pg::kKC - 1) / pg::kKC;
  a.ntiles_n = (N + NT - 1) / NT;
  a.mtiles_per_b = (ln + 127) / 128;
  if (fn == FN_NONE) return by_layout<128>(a, act_layout, out_layout, sms, s);
  if (act_layout == pg::ACT_CH && out_layout == pg::OUT_ROW) {          // GELU prologue (MLP fc2 forward)
    if (fn == FN_GELU_TANH) return go<128, pg::ACT_CH, pg::OUT_ROW, FN_GELU_TANH>(a, sms, s, K_PROJ_GEMM_GELU);
    if (fn == FN_GELU_ERF) return go<128, pg::ACT_CH, pg::OUT_ROW, FN_GELU_ERF>(a, sms, s, K_PROJ_GEMM_GELU);
  }
  if (act_layout == pg::ACT_ROW && out_layout == pg::OUT_CH) {          // GELU-gradient epilogue (MLP fc2 input gradient)
    if (fn == FN_GELU_TANH) return go<128, pg::ACT_ROW, pg::OUT_CH, FN_GELU_TANH>(a, sms, s, K_PROJ_GEMM_DGELU);
    if (fn == FN_GELU_ERF) return go<128, pg::ACT_ROW, pg::OUT_CH, FN_GELU_ERF>(a, sms, s, K_PROJ_GEMM_DGELU);
  }
  return cudaErrorInvalidValue;
}


// weight gradient: dW (M, N) [or (N, M) when transposed_out] = sum_{b,pos} X[b][m][pos] Y[b][pos][n]
void proj_wgrad_plan(int M, int N, int sms, int* mtiles, int* ntiles, int* splits) {
  *mtiles = (M + 127) / 128;
  *ntiles = (N + 127) / 128;
  int s = sms / (*mtiles * *ntiles);
  *splits = s < 1 ? 1 : s;
}

size_t proj_wgrad_scratch_bytes(int M, int N) {
  int dev = 0, sms = 132, mt, nt, sp;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  proj_wgrad_plan(M, N, sms, &mt, &nt, &sp);
  return (size_t)sp * M * N * sizeof(float);
}

cudaError_t launch_proj_wgrad(const float* X, const float* Y, const float* fir, float* dW, int transposed_out, float beta,
                              int B, int L, int M, int N, float* part, cudaStream_t s, int fn) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  wg::Args a;
  a.X = X; a.Y = Y; a.fir = fir; a.part = part; a.zero = 0; a.B = B; a.L = L; a.M = M; a.N = N;
  a.chunks_per_b = (L + 31) / 32;
  proj_wgrad_plan(M, N, sms, &a.mtiles, &a.ntiles, &a.splits);
  const long long total_chunks = (long long)B * a.chunks_per_b;
  if (a.splits > total_chunks) a.splits = (int)total_chunks;
  a.vec = (L % 4 == 0) && (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15u) == 0;
  CUtensorMap tmx, tmy;
  memset(&tmx, 0, sizeof(tmx)); memset(&tmy, 0, sizeof(tmy));
  if (a.vec) {
    // X (B, M, L): box 36 positions x 128 rows;  Y (B, L, N): box 128 columns x 32 positions
    const bool ok = make_tmap3(&tmx, X, (unsigned long long)L, (unsigned long long)M, (unsigned long long)B, 36, 128) &&
                    make_tmap3(&tmy, Y, (unsigned long long)N, (unsigned long long)L, (unsigned long long)B, 128, 32);
    if (!ok) a.vec = 0;                  // no driver entry point / unencodable shape: the producer warp stages by hand
  }
  auto kern = fn == FN_GELU_TANH ? wg::wgrad_kernel<FN_GELU_TANH>
            : fn == FN_GELU_ERF  ? wg::wgrad_kernel<FN_GELU_ERF> : wg::wgrad_kernel<FN_NONE>;
  if (fn != FN_NONE && (fir || (fn != FN_GELU_TANH && fn != FN_GELU_ERF))) return cudaErrorInvalidValue;
  const int kind = fn == FN_NONE ? K_PROJ_WGRAD : K_PROJ_WGRAD_GELU;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg::kSmem);
  if (e != cudaSuccess) return e;
  prof_begin(kind, s);
  kern<<<a.mtiles * a.ntiles * a.splits, wg::kThreads, wg::kSmem, s>>>(a, tmx, tmy);
  prof_end(kind, s);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const size_t total = (size_t)M * N;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 2 * sms) blocks = 2 * sms;
  prof_begin(kind, s);
  wg::wgrad_reduce_kernel<<<blocks, 256, 0, s>>>(part, dW, a.splits, M, N, transposed_out, beta);
  prof_end(kind, s);
  return cudaGetLastError();
}

}  // namespace hy
