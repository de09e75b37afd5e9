// C ABI of libhyena_b200.so (include/hyena_b200.h): argument checks, workspace carving, row-group
// scheduling of the three FFT passes.  No torch types; PyTorch hands in raw device pointers.
#include <atomic>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/hyena_b200.h"
#include "launch.h"

namespace hy {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

// ---- optional per-launch event timing (bench.py's roofline leg); off by default
struct ProfRec { int kind; cudaEvent_t e0, e1; };
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;            // records of the current profiling window
static std::vector<cudaEvent_t> g_ev_pool;     // recycled events
static thread_local cudaEvent_t g_cur_e0 = nullptr;

static cudaEvent_t get_event() {
  if (!g_ev_pool.empty()) { cudaEvent_t e = g_ev_pool.back(); g_ev_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
// a stream being captured into a CUDA graph gets no timing events: they would become graph nodes, and the pooled events
// would be recycled while the graph still records them
static bool capturing(cudaStream_t s) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  return cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone;
}
void prof_begin(int kind, cudaStream_t s) {
  (void)kind;
  if (!g_prof_on || capturing(s)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_cur_e0 = get_event();
  cudaEventRecord(g_cur_e0, s);
}
void prof_end(int kind, cudaStream_t s) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (!g_prof_on || !g_cur_e0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEvent_t e1 = get_event();
  cudaEventRecord(e1, s);
  g_prof.push_back({kind, g_cur_e0, e1});
  g_cur_e0 = nullptr;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int api_fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
#define HY_CUDA(expr)                                                                        \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) return fail("%s failed: %s", #expr, cudaGetErrorString(_e));      \
  } while (0)
#define HY_CHECK(cond, ...) \
  do { if (!(cond)) return fail(__VA_ARGS__); } while (0)

// ---------------------------------------------------------------- per-device twiddle tables
struct DevTables { float2* tw1024 = nullptr; float2* twlo = nullptr; };
static DevTables g_tables[64];
static std::mutex g_mu;

static int get_twiddles(cudaStream_t s, Twiddles* out) {
  int dev = -1;
  HY_CUDA(cudaGetDevice(&dev));
  HY_CHECK(dev >= 0 && dev < 64, "unsupported device ordinal %d", dev);
  std::lock_guard<std::mutex> lk(g_mu);
  DevTables& t = g_tables[dev];
  if (!t.tw1024) {
    float2* mem = nullptr;
    HY_CUDA(cudaMalloc(&mem, 2 * 1024 * sizeof(float2)));
    HY_CUDA(launch_twiddle_init(mem, mem + 1024, s));
    // later calls may come on other streams: make the table visible to all of them
    HY_CUDA(cudaStreamSynchronize(s));
    t.tw1024 = mem;
    t.twlo = mem + 1024;
  }
  out->tw1024 = t.tw1024;
  out->twlo = t.twlo;
  return 0;
}

// ---------------------------------------------------------------- geometry
static int log_m_for(int L) {         // M = 2^logM >= max(L, 1024)
  int lg = 10;
  while (((size_t)1 << lg) < (size_t)L) ++lg;
  return lg;
}
// Row length: 1024 points, one warp per row.
static int pick_log_m2(int) { return 10; }
static size_t row_bytes(int L) { return ((size_t)1 << log_m_for(L)) * sizeof(float2); }

static size_t group_budget_bytes() {
  // scratch rows in flight per launch group: with separate kernels per pass the scratch does not survive in L2 anyway,
  // and many waves per launch win, so the default lets a whole (B=1, D=256, L=2^20) operator go in one launch per pass
  static size_t v = 0;
  if (!v) {
    const char* e = getenv("HYENA_B200_GROUP_MB");
    long mb = e ? atol(e) : 2048;
    if (mb < 1) mb = 1;
    v = (size_t)mb << 20;
  }
  return v;
}

// channels per group given the bytes available for ONE scratch array holding all batches of a channel
static int channels_per_group(size_t bytes_for_A, int B, int D, int L) {
  size_t per_ch = row_bytes(L) * (size_t)B;
  size_t n = bytes_for_A / per_ch;
  if (n > (size_t)D) n = D;
  size_t cap = 65535 / (size_t)B;
  if (n > cap) n = cap;
  return (int)n;
}

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
// a decode history of element type T: one element, and the 4 positions the vector loads and the shift move at once
template <class T> static bool elem_aligned(const T* p) { return reinterpret_cast<uintptr_t>(p) % sizeof(T) == 0; }
template <class T> static bool hist_aligned(const T* p) { return reinterpret_cast<uintptr_t>(p) % (4 * sizeof(T)) == 0; }
template <class T> constexpr bool kFp32 = std::is_same<T, float>::value;
template <class T> constexpr const char* kAlignH = kFp32<T> ? "h must be 16-byte aligned" : "h must be 8-byte aligned";
template <class T> constexpr const char* kAlignKH =
    kFp32<T> ? "k and h must be 16-byte aligned" : "k must be 16-byte aligned and h 8-byte aligned";

struct Carve { float2* A; float2* A2; float2* A3; int nch; };

// backward needs A and A2 (B rows per channel each) and A3 (1 row per channel)
static int carve(void* ws, size_t ws_bytes, int B, int D, int L, bool backward, Carve* c) {
  HY_CHECK(ws != nullptr && aligned8(ws), "workspace must be a non-null 8-byte aligned device pointer");
  const size_t rb = row_bytes(L);
  const size_t per_ch = backward ? rb * (2 * (size_t)B + 1) : rb * (size_t)B;
  HY_CHECK(ws_bytes >= per_ch, "workspace too small: %zu bytes given, %zu needed (hyena_b200_workspace_min_bytes)",
           ws_bytes, per_ch);
  size_t n = ws_bytes / per_ch;
  if (n > (size_t)D) n = D;
  size_t cap = 65535 / (size_t)B;
  if (n > cap) n = cap;
  c->nch = (int)n;
  c->A = reinterpret_cast<float2*>(ws);
  c->A2 = backward ? c->A + (rb / sizeof(float2)) * (size_t)B * n : nullptr;
  c->A3 = backward ? c->A2 + (rb / sizeof(float2)) * (size_t)B * n : nullptr;
  return 0;
}

static int check_shape(int B, int D, int L) {
  HY_CHECK(B >= 1 && D >= 1 && L >= 1, "bad shape B=%d D=%d L=%d", B, D, L);
  HY_CHECK(L <= (1 << 20), "sequence length %d exceeds the supported maximum %d", L, 1 << 20);
  HY_CHECK(B <= 65535, "batch %d too large", B);
  return 0;
}

static PassArgs base_args(int B, int D, int L, const Twiddles& T) {
  PassArgs a;
  memset(&a, 0, sizeof(a));
  const int logM = log_m_for(L);
  a.L = L; a.logM2 = pick_log_m2(logM); a.logM1 = logM - a.logM2; a.B = B; a.D = D; a.T = T;
  a.scale = 1.0f / (4.0f * (float)((size_t)1 << logM));
  return a;
}

}  // namespace hy

using namespace hy;

extern "C" {

HY_API int hyena_b200_abi_version(void) { return HYENA_B200_ABI_VERSION; }
HY_API const char* hyena_b200_last_error(void) { return g_err; }
HY_API unsigned long long hyena_b200_launch_count(void) { return g_launches.load(); }
HY_API int hyena_b200_max_seqlen(void) { return 1 << 20; }

HY_API int hyena_b200_profile_begin(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto& r : g_prof) { g_ev_pool.push_back(r.e0); g_ev_pool.push_back(r.e1); }
  g_prof.clear();
  g_prof_on = true;
  return 0;
}

HY_API int hyena_b200_profile_end(double* ms_by_kind, unsigned long long* launches_by_kind, int n) {
  HY_CHECK(ms_by_kind && launches_by_kind && n >= K_COUNT, "profile_end needs arrays of >= %d entries", K_COUNT);
  HY_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = false;
  for (int i = 0; i < n; ++i) { ms_by_kind[i] = 0.0; launches_by_kind[i] = 0; }
  for (auto& r : g_prof) {
    float ms = 0.f;
    HY_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
    ms_by_kind[r.kind] += ms;
    launches_by_kind[r.kind] += 1;
    g_ev_pool.push_back(r.e0); g_ev_pool.push_back(r.e1);
  }
  g_prof.clear();
  return 0;
}

HY_API const char* hyena_b200_kind_name(int kind) {
  static const char* names[K_COUNT] = {
      "col_fwd<filter>", "col_fwd<gate>", "col_fwd<dc>", "col_fwd<plain>",
      "col_inv<conv_fwd>", "col_inv<bwd_dg>", "col_inv<dk>", "col_inv<plain_fwd>", "col_inv<plain_bwd>",
      "row_pass<filter>", "row_pass<conv_fwd>", "row_pass<conv_bwd>",
      "short_conv_bwd", "twiddle_init", "filter_tc_prep", "filter_tc_fwd", "filter_tc_bwd", "filter_tc_red",
      "spectrum_convert", "proj_prep", "proj_gemm", "proj_wgrad", "add_layer_norm", "filter_extra",
      "proj_gemm<gelu>", "proj_gemm<dgelu>", "proj_wgrad<gelu>", "decode_hist", "decode_step",
      "decode_extend_hist", "decode_extend_dot", "decode_extend_combine", "decode_win_step"};
  return (kind >= 0 && kind < K_COUNT) ? names[kind] : "?";
}

HY_API int hyena_b200_kind_count(void) { return K_COUNT; }

HY_API size_t hyena_b200_spectrum_elems(int L) { return L < 1 ? 0 : ((size_t)1 << log_m_for(L)); }

HY_API size_t hyena_b200_workspace_min_bytes(int B, int D, int L, int backward) {
  (void)D;
  if (B < 1 || L < 1) return 0;
  return backward ? row_bytes(L) * (2 * (size_t)B + 1) : row_bytes(L) * (size_t)B;
}

HY_API size_t hyena_b200_workspace_bytes(int B, int D, int L, int backward) {
  if (B < 1 || L < 1 || D < 1) return 0;
  int nch = channels_per_group(group_budget_bytes(), B, D, L);
  if (nch < 1) nch = 1;
  return hyena_b200_workspace_min_bytes(B, D, L, backward) * (size_t)nch;
}

// tensor-core filter path: scratch, grow-only, one per (device, stream, use): two operators driven from different streams
// never share it (the prep kernel of one would overwrite the images the other's wgmma kernel is still reading).
// Uses: 0 = the tf32 hi/lo weight images (~0.3 MB), 1 = stage 2's [zT; 1] and partial sums (~40 MB at L = 2^20)
static int get_filter_buf(int use, size_t need, cudaStream_t stream, float** out) {
  int dev = -1;
  HY_CUDA(cudaGetDevice(&dev));
  HY_CHECK(dev >= 0 && dev < 64, "unsupported device ordinal %d", dev);
  std::lock_guard<std::mutex> lk(g_mu);
  struct Buf { float* p = nullptr; size_t n = 0; };
  static std::map<std::tuple<int, cudaStream_t, int>, Buf> bufs;
  Buf& b = bufs[std::make_tuple(dev, stream, use)];
  if (b.n < need) {
    if (b.p) { HY_CUDA(cudaStreamSynchronize(stream)); HY_CUDA(cudaFree(b.p)); b.p = nullptr; b.n = 0; }
    HY_CUDA(cudaMalloc(&b.p, need));
    b.n = need;
  }
  *out = b.p;
  return 0;
}
static int get_wimg(int D, cudaStream_t stream, float** out) { return get_filter_buf(0, filter_tc_wimg_bytes(D), stream, out); }

static int fill_filter_params(FilterParams* P, const float* z, int z_stride, const float* t, const float* W0,
                              const float* b0, const float* W1, const float* b1, const float* W2, const float* b2,
                              const float* W3, const float* freq, const float* deltas, float shift, int modulate,
                              int L, int E, int N, int D) {
  HY_CHECK(N == kFN, "filter_order %d not supported (this build handles %d)", N, kFN);
  HY_CHECK(E >= 3 && E < kMaxE && (E & 1), "emb_dim %d not supported (odd, 3..%d)", E, kMaxE - 1);
  HY_CHECK(L >= 1 && D >= 1, "bad filter shape L=%d D=%d", L, D);
  HY_CHECK(z && t && W0 && b0 && W1 && b1 && W2 && b2 && W3 && freq && deltas, "null filter parameter");
  HY_CHECK((reinterpret_cast<uintptr_t>(W3) & 15u) == 0, "W3 must be 16-byte aligned");
  P->z = z; P->t = t; P->W0 = W0; P->b0 = b0; P->W1 = W1; P->b1 = b1; P->W2 = W2; P->b2 = b2; P->W3 = W3;
  P->freq = freq; P->deltas = deltas; P->shift = shift; P->modulate = modulate;
  P->L = L; P->E = E; P->D = D; P->z_stride = z_stride;
  return 0;
}

HY_API int hyena_b200_filter_fwd(const float* z, int z_stride, const float* t, const float* W0, const float* b0,
                          const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                          const float* freq, const float* deltas, float shift, int modulate, int L, int E, int N,
                          int D, float* k_out, void* stream) {
  FilterParams P;
  if (fill_filter_params(&P, z, z_stride, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, E, N, D))
    return 1;
  HY_CHECK(k_out, "null output");
  float* wimg = nullptr;
  if (get_wimg(D, (cudaStream_t)stream, &wimg)) return 1;
  HY_CUDA(launch_filter_fwd_tc(P, wimg, k_out, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_filter_bwd_stage1(const float* z, int z_stride, const float* t, const float* W0, const float* b0,
                                 const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                                 const float* freq, const float* deltas, float shift, int modulate, int L, int E,
                                 int N, int D, const float* dk, float* dh, float* scratch, void* stream) {
  FilterParams P;
  if (fill_filter_params(&P, z, z_stride, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, E, N, D))
    return 1;
  HY_CHECK(dk && dh && scratch && ((reinterpret_cast<uintptr_t>(scratch) & 15u) == 0), "null or misaligned pointer");
  float* wimg = nullptr;
  if (get_wimg(D, (cudaStream_t)stream, &wimg)) return 1;
  HY_CUDA(launch_filter_bwd_tc(P, wimg, dk, dh, scratch, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_filter_bwd_stage2(const float* dh, const float* scratch, const float* zT, float* dW0, float* db0,
                                 float* dW1, float* db1, float* dW2, float* db2, float* dW3, float* dfreq, int L,
                                 int E, int D, void* stream) {
  HY_CHECK(dh && scratch && zT && dW0 && db0 && dW1 && db1 && dW2 && db2 && dW3 && dfreq, "null pointer");
  HY_CHECK(D >= 1 && D <= 256 && E >= 1 && E <= 8 && L >= 1, "fused filter reduction handles D <= 256, E <= 8 (got D=%d E=%d)", D, E);
  HY_CHECK((reinterpret_cast<uintptr_t>(dh) & 15u) == 0 && (reinterpret_cast<uintptr_t>(scratch) & 15u) == 0 &&
               (reinterpret_cast<uintptr_t>(zT) & 15u) == 0, "misaligned pointer");
  float* work = nullptr;
  if (get_filter_buf(1, filter_red_work_bytes(L, D, E), (cudaStream_t)stream, &work)) return 1;
  RedLaunch r{dh, scratch, zT, dW0, db0, dW1, db1, dW2, db2, dW3, dfreq, L, D, E};
  HY_CUDA(launch_filter_stage2(r, work, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_filter_spectrum(const float* k, float* kspec, int D, int L, void* workspace, size_t workspace_bytes,
                               void* stream) {
  if (check_shape(1, D, L)) return 1;
  HY_CHECK(k && kspec && aligned8(kspec), "null or misaligned pointer");
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, 1, D, L, false, &c)) return 1;
  PassArgs a = base_args(1, D, L, T);
  a.A = c.A; a.src = k; a.kspec_out = reinterpret_cast<float2*>(kspec);
  a.vec = ((L & 1) == 0) && aligned8(k);
  for (int c0 = 0; c0 < D; c0 += c.nch) {
    const int n = (D - c0 < c.nch) ? D - c0 : c.nch;
    a.c0 = c0;
    HY_CUDA(launch_col_fwd(COL_FILTER, a, n, s));
    HY_CUDA(launch_row_pass(ROW_FILTER, a, n, s));
  }
  return 0;
}

/* filter = rfft(k, fft_size) (H, fft_size/2+1) complex64, natural order, unnormalised -> packed kspec (H, M).
 * k_scratch (H*L floats) is used only when fft_size < 2M (sequences shorter than the minimum transform). */
HY_API int hyena_b200_spectrum_from_rfft(const float* filter, int fft_size, float* kspec, float* k_scratch, int H, int L,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(1, H, L)) return 1;
  HY_CHECK(filter && kspec && aligned8(filter) && aligned8(kspec), "null or misaligned pointer");
  HY_CHECK(fft_size >= 16 && (fft_size & (fft_size - 1)) == 0 && L <= fft_size / 2,
           "fft_size %d must be a power of two >= 16 with L = %d <= fft_size/2 (fftconv.cpp:114-115)", fft_size, L);
  cudaStream_t s = (cudaStream_t)stream;
  const int logM = log_m_for(L);
  const int logM2 = pick_log_m2(logM), logM1 = logM - logM2;
  if ((size_t)fft_size == ((size_t)2 << logM)) {
    HY_CUDA(launch_rfft_to_packed(reinterpret_cast<const float2*>(filter), reinterpret_cast<float2*>(kspec), H, logM, logM1, s));
    return 0;
  }
  HY_CHECK((size_t)fft_size < ((size_t)2 << logM), "fft_size %d larger than the transform of L = %d", fft_size, L);
  HY_CHECK(k_scratch, "k_scratch is required when fft_size < 2 * spectrum_elems(L)");
  HY_CUDA(launch_rfft_to_time_small(reinterpret_cast<const float2*>(filter), k_scratch, H, L, fft_size, s));
  return hyena_b200_filter_spectrum(k_scratch, kspec, H, L, workspace, workspace_bytes, stream);
}

/* dk (H, L) time domain -> dfilter (H, fft_size/2+1) complex64 with irfft(dfilter, n=fft_size, norm='forward')[:L] == dk
 * (the convention of csrc/fftconv/fftconv.cpp:235 consumed by src/ops/fftconv.py:98).  kspec_scratch: (H, M) complex. */
HY_API int hyena_b200_spectrum_to_rfft(const float* dk, int fft_size, float* dfilter, float* kspec_scratch, int H, int L,
                                void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(1, H, L)) return 1;
  HY_CHECK(dk && dfilter && aligned8(dfilter), "null or misaligned pointer");
  HY_CHECK(fft_size >= 16 && (fft_size & (fft_size - 1)) == 0 && L <= fft_size / 2,
           "fft_size %d must be a power of two >= 16 with L = %d <= fft_size/2", fft_size, L);
  cudaStream_t s = (cudaStream_t)stream;
  const int logM = log_m_for(L);
  const int logM2 = pick_log_m2(logM), logM1 = logM - logM2;
  const float scale = 1.0f / (float)fft_size;
  if ((size_t)fft_size == ((size_t)2 << logM)) {
    HY_CHECK(kspec_scratch && aligned8(kspec_scratch), "kspec_scratch is required");
    if (hyena_b200_filter_spectrum(dk, kspec_scratch, H, L, workspace, workspace_bytes, stream)) return 1;
    HY_CUDA(launch_packed_to_rfft(reinterpret_cast<const float2*>(kspec_scratch), reinterpret_cast<float2*>(dfilter), H, logM,
                                  logM1, scale, s));
    return 0;
  }
  HY_CHECK((size_t)fft_size < ((size_t)2 << logM), "fft_size %d larger than the transform of L = %d", fft_size, L);
  HY_CUDA(launch_time_to_rfft_small(dk, reinterpret_cast<float2*>(dfilter), H, L, fft_size, scale, s));
  return 0;
}

// the three forward passes of core_fwd; row_start non-null: the left-padded modes (core_fwd_rows), seg_base non-null as
// well: the packed modes (core_fwd_packed, channel stride `total`); the same launch sequence
static int core_fwd_run(const float* p, const float* in_bias, const float* sw, const float* sb, const float* kspec,
                        const float* fbias, float* y_pre, float* c_save, float* gspec_save, const int* row_start, int B,
                        int D, int L, void* workspace, size_t workspace_bytes, void* stream,
                        const long long* seg_base = nullptr, long long total = 0, const int* out_start = nullptr) {
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, D, L, false, &c)) return 1;
  PassArgs a = base_args(B, D, L, T);
  a.A = c.A; a.kspec = reinterpret_cast<const float2*>(kspec);
  a.p = p; a.in_bias = in_bias; a.sw = sw; a.sb = sb; a.fbias = fbias; a.out = y_pre; a.out2 = c_save;
  a.gspec = reinterpret_cast<float2*>(gspec_save);
  a.row_start = row_start;
  a.vec = ((L & 1) == 0) && aligned8(p) && aligned8(y_pre) && (!c_save || aligned8(c_save));
  a.stage = ((L & 3) == 0) && aligned16(p);
  int col_mode = row_start ? COL_GATE_ROWS : COL_GATE, inv_mode = row_start ? INV_CONV_FWD_ROWS : INV_CONV_FWD;
  if (seg_base) {            // packed: scalar accesses to p and y_pre; vec covers c_save only
    a.seg_base = seg_base; a.cstride = total;
    a.vec = ((L & 1) == 0) && (!c_save || aligned8(c_save));
    a.stage = 0;
    col_mode = COL_GATE_PACKED; inv_mode = INV_CONV_FWD_PACKED;
    if (out_start) { a.out_start = out_start; inv_mode = INV_CONV_FWD_WIN; }   // windows: COL_GATE_PACKED reads them as is
  }
  for (int c0 = 0; c0 < D; c0 += c.nch) {
    const int n = (D - c0 < c.nch) ? D - c0 : c.nch;
    a.c0 = c0;
    HY_CUDA(launch_col_fwd(col_mode, a, n * B, s));
    HY_CUDA(launch_row_pass(ROW_CONV_FWD, a, n * B, s));
    HY_CUDA(launch_col_inv(inv_mode, a, n * B, s));
  }
  return 0;
}

HY_API int hyena_b200_core_fwd(const float* p, const float* in_bias, const float* sw, const float* sb, const float* kspec,
                        const float* fbias, float* y_pre, float* c_save, float* gspec_save, int B, int D, int L,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(p && sw && sb && kspec && fbias && y_pre, "null pointer");
  return core_fwd_run(p, in_bias, sw, sb, kspec, fbias, y_pre, c_save, gspec_save, nullptr, B, D, L, workspace,
                      workspace_bytes, stream);
}

HY_API int hyena_b200_core_fwd_rows(const float* p, const float* in_bias, const float* sw, const float* sb,
                                    const float* kspec, const float* fbias, float* y_pre, float* c_save, float* gspec_save,
                                    const int* row_start, int B, int D, int L, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(p && sw && sb && kspec && fbias && y_pre && row_start, "null pointer");
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && aligned4(fbias) && aligned4(y_pre) && aligned4(row_start) &&
               (!in_bias || aligned4(in_bias)) && (!c_save || aligned4(c_save)),
           "misaligned pointer: p, in_bias, sw, sb, fbias, y_pre, c_save and row_start must be 4-byte aligned");
  HY_CHECK(aligned8(kspec) && (!gspec_save || aligned8(gspec_save)), "misaligned pointer: kspec and gspec_save must be "
           "8-byte aligned");
  return core_fwd_run(p, in_bias, sw, sb, kspec, fbias, y_pre, c_save, gspec_save, row_start, B, D, L, workspace,
                      workspace_bytes, stream);
}

// the backward passes of core_bwd; row_start non-null: the left-padded modes (core_bwd_rows), seg_base non-null as well:
// the packed modes (core_bwd_packed: dp == NULL, ds_scratch packed); the same launch sequence
static int core_bwd_run(const float* dy_pre, const float* p, const float* in_bias, const float* sw, const float* sb,
                        const float* kspec, const float* fbias, const float* c_saved, const float* gspec_saved, float* dp,
                        float* dk, float* dsw, float* dsb, float* dfbias, float* d_in_bias, float* ds_scratch,
                        const int* row_start, int B, int D, int L, void* workspace, size_t workspace_bytes, void* stream,
                        const long long* seg_base = nullptr, long long total = 0) {
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, D, L, true, &c)) return 1;
  PassArgs a = base_args(B, D, L, T);
  a.kspec = reinterpret_cast<const float2*>(kspec);
  a.p = p; a.in_bias = in_bias; a.sw = sw; a.sb = sb; a.fbias = fbias;
  a.row_start = row_start;
  int dc_mode = row_start ? COL_DC_ROWS : COL_DC, gate_mode = row_start ? COL_GATE_ROWS : COL_GATE,
      dg_mode = row_start ? INV_BWD_DG_ROWS : INV_BWD_DG;
  a.vec = ((L & 1) == 0) && aligned8(p) && aligned8(dy_pre) && aligned8(c_saved) && aligned8(dk) &&
          aligned8(ds_scratch);
  a.stage = ((L & 3) == 0) && aligned16(p) && aligned16(dy_pre) && aligned16(c_saved);
  if (seg_base) {            // packed: scalar accesses to p, dy_pre and ds; vec covers c_saved and dk only
    a.seg_base = seg_base; a.cstride = total;
    a.vec = ((L & 1) == 0) && aligned8(c_saved) && aligned8(dk);
    a.stage = 0;
    dc_mode = COL_DC_PACKED; gate_mode = COL_GATE_PACKED; dg_mode = INV_BWD_DG_PACKED;
  }
  for (int c0 = 0; c0 < D; c0 += c.nch) {
    const int n = (D - c0 < c.nch) ? D - c0 : c.nch;
    a.c0 = c0; a.B = B;
    a.A2 = c.A2; a.A3 = c.A3;
    a.A = c.A; a.src = dy_pre;
    HY_CUDA(launch_col_fwd(dc_mode, a, n * B, s));       // A  <- columns of dc = dy_pre * x0
    a.gspec = const_cast<float2*>(reinterpret_cast<const float2*>(gspec_saved));
    if (!gspec_saved) {
      a.A = c.A2;
      HY_CUDA(launch_col_fwd(gate_mode, a, n * B, s));   // A2 <- columns of g = v * x1 (recomputed)
    }
    a.A = c.A;
    // (the 128-thread batch-1 kernel exists for 1024-point rows only)
    HY_CUDA(launch_row_pass((B == 1 && gspec_saved && a.logM2 == 10) ? ROW_CONV_BWD1 : ROW_CONV_BWD, a, n, s));   // A <- rows of dg, A3 <- rows of dk
    a.src = dy_pre; a.src2 = c_saved; a.out2 = ds_scratch; a.red = dfbias; a.dsw = dsw; a.dsb = dsb;
    HY_CUDA(launch_col_inv(dg_mode, a, n * B, s));
    a.B = 1; a.out = dk;
    HY_CUDA(launch_col_inv(INV_DK, a, n, s));
  }
  // pass 3 already accumulated dsw / dsb from the operand windows it had staged: no second read of p here.
  // dp == NULL: the caller consumes ds directly (hyena_b200_proj_gemm / proj_wgrad apply the transposed short filter on
  // the fly and d in_proj.bias follows from dsb and two edge samples), so dp never exists in HBM.
  if (dp) {
    ShortBwdArgs sa{ds_scratch, nullptr, in_bias, sw, dp, dsw, dsb, d_in_bias, L, 3 * D, a.vec && aligned8(dp), row_start,
                    nullptr, 0};
    HY_CUDA(launch_short_bwd(sa, B, s));
  }
  return 0;
}

HY_API int hyena_b200_core_bwd(const float* dy_pre, const float* p, const float* in_bias, const float* sw, const float* sb,
                        const float* kspec, const float* fbias, const float* c_saved, const float* gspec_saved,
                        float* dp, float* dk, float* dsw, float* dsb, float* dfbias, float* d_in_bias,
                        float* ds_scratch, int B, int D, int L, void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(dy_pre && p && sw && sb && kspec && fbias && c_saved && dk && dsw && dsb && dfbias && ds_scratch,
           "null pointer");
  return core_bwd_run(dy_pre, p, in_bias, sw, sb, kspec, fbias, c_saved, gspec_saved, dp, dk, dsw, dsb, dfbias, d_in_bias,
                      ds_scratch, nullptr, B, D, L, workspace, workspace_bytes, stream);
}

HY_API int hyena_b200_core_bwd_rows(const float* dy_pre, const float* p, const float* in_bias, const float* sw,
                                    const float* sb, const float* kspec, const float* fbias, const float* c_saved,
                                    const float* gspec_saved, float* dp, float* dk, float* dsw, float* dsb, float* dfbias,
                                    float* d_in_bias, float* ds_scratch, const int* row_start, int B, int D, int L,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(dy_pre && p && sw && sb && kspec && fbias && c_saved && dk && dsw && dsb && dfbias && ds_scratch && row_start,
           "null pointer");
  HY_CHECK(aligned4(dy_pre) && aligned4(p) && aligned4(sw) && aligned4(sb) && aligned4(fbias) && aligned4(c_saved) &&
               aligned4(dk) && aligned4(dsw) && aligned4(dsb) && aligned4(dfbias) && aligned4(ds_scratch) &&
               aligned4(row_start) && (!in_bias || aligned4(in_bias)) && (!dp || aligned4(dp)) &&
               (!d_in_bias || aligned4(d_in_bias)),
           "misaligned pointer: every float operand and row_start must be 4-byte aligned");
  HY_CHECK(aligned8(kspec) && (!gspec_saved || aligned8(gspec_saved)), "misaligned pointer: kspec and gspec_saved must be "
           "8-byte aligned");
  return core_bwd_run(dy_pre, p, in_bias, sw, sb, kspec, fbias, c_saved, gspec_saved, dp, dk, dsw, dsb, dfbias, d_in_bias,
                      ds_scratch, row_start, B, D, L, workspace, workspace_bytes, stream);
}

// the arguments every packed entry point shares: B rows of length L over a packed tensor of `total` positions
static int check_packed(const long long* seg_base, const int* row_start, long long total, int B, int D, int L) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(total >= 1, "bad packed length total=%lld", total);
  HY_CHECK(seg_base && row_start, "null pointer");
  HY_CHECK(aligned8(seg_base) && aligned4(row_start), "misaligned pointer: seg_base must be 8-byte and row_start 4-byte "
           "aligned");
  return 0;
}

HY_API int hyena_b200_core_fwd_packed(const float* p, const float* in_bias, const float* sw, const float* sb,
                                      const float* kspec, const float* fbias, float* y_pre, float* c_save,
                                      float* gspec_save, const long long* seg_base, const int* row_start, long long total,
                                      int B, int D, int L, void* workspace, size_t workspace_bytes, void* stream) {
  if (check_packed(seg_base, row_start, total, B, D, L)) return 1;
  HY_CHECK(p && sw && sb && kspec && fbias && y_pre, "null pointer");
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && aligned4(fbias) && aligned4(y_pre) &&
               (!in_bias || aligned4(in_bias)) && (!c_save || aligned4(c_save)),
           "misaligned pointer: p, in_bias, sw, sb, fbias, y_pre and c_save must be 4-byte aligned");
  HY_CHECK(aligned8(kspec) && (!gspec_save || aligned8(gspec_save)), "misaligned pointer: kspec and gspec_save must be "
           "8-byte aligned");
  return core_fwd_run(p, in_bias, sw, sb, kspec, fbias, y_pre, c_save, gspec_save, row_start, B, D, L, workspace,
                      workspace_bytes, stream, seg_base, total);
}

// the guards both window entry points share (check_packed, plus out_start)
static int check_windows(const long long* seg_base, const int* row_start, const int* out_start, long long total, int B,
                         int D, int L) {
  if (check_packed(seg_base, row_start, total, B, D, L)) return 1;
  HY_CHECK(out_start && aligned4(out_start), "null or misaligned pointer: out_start must be 4-byte aligned");
  return 0;
}

HY_API int hyena_b200_core_fwd_windows(const float* p, const float* in_bias, const float* sw, const float* sb,
                                       const float* kspec, const float* fbias, float* y_pre, const long long* seg_base,
                                       const int* row_start, const int* out_start, long long total, int B, int D, int L,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  if (check_windows(seg_base, row_start, out_start, total, B, D, L)) return 1;
  HY_CHECK(p && sw && sb && kspec && fbias && y_pre, "null pointer");
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && aligned4(fbias) && aligned4(y_pre) &&
               (!in_bias || aligned4(in_bias)),
           "misaligned pointer: p, in_bias, sw, sb, fbias and y_pre must be 4-byte aligned");
  HY_CHECK(aligned8(kspec), "misaligned pointer: kspec must be 8-byte aligned");
  return core_fwd_run(p, in_bias, sw, sb, kspec, fbias, y_pre, nullptr, nullptr, row_start, B, D, L, workspace,
                      workspace_bytes, stream, seg_base, total, out_start);
}

HY_API int hyena_b200_core_bwd_packed(const float* dy_pre, const float* p, const float* in_bias, const float* sw,
                                      const float* sb, const float* kspec, const float* fbias, const float* c_saved,
                                      const float* gspec_saved, float* dk, float* dsw, float* dsb, float* dfbias,
                                      float* ds, const long long* seg_base, const int* row_start, long long total, int B,
                                      int D, int L, void* workspace, size_t workspace_bytes, void* stream) {
  if (check_packed(seg_base, row_start, total, B, D, L)) return 1;
  HY_CHECK(dy_pre && p && sw && sb && kspec && fbias && c_saved && dk && dsw && dsb && dfbias && ds, "null pointer");
  HY_CHECK(aligned4(dy_pre) && aligned4(p) && aligned4(sw) && aligned4(sb) && aligned4(fbias) && aligned4(c_saved) &&
               aligned4(dk) && aligned4(dsw) && aligned4(dsb) && aligned4(dfbias) && aligned4(ds) &&
               (!in_bias || aligned4(in_bias)),
           "misaligned pointer: every float operand must be 4-byte aligned");
  HY_CHECK(aligned8(kspec) && (!gspec_saved || aligned8(gspec_saved)), "misaligned pointer: kspec and gspec_saved must be "
           "8-byte aligned");
  return core_bwd_run(dy_pre, p, in_bias, sw, sb, kspec, fbias, c_saved, gspec_saved, nullptr, dk, dsw, dsb, dfbias,
                      nullptr, ds, row_start, B, D, L, workspace, workspace_bytes, stream, seg_base, total);
}

HY_API int hyena_b200_short_bwd_packed(const float* ds, const float* sw, float* dp, float* d_in_bias,
                                       const long long* seg_base, const int* row_start, long long total, int B, int C3,
                                       int L, void* stream) {
  if (check_packed(seg_base, row_start, total, B, C3, L)) return 1;
  HY_CHECK(ds && sw && dp, "null pointer");
  HY_CHECK(aligned4(ds) && aligned4(sw) && aligned4(dp) && (!d_in_bias || aligned4(d_in_bias)),
           "misaligned pointer: ds, sw, dp and d_in_bias must be 4-byte aligned");
  ShortBwdArgs sa{ds, nullptr, nullptr, sw, dp, nullptr, nullptr, d_in_bias, L, C3, 0, row_start, seg_base, total};
  HY_CUDA(launch_short_bwd(sa, B, (cudaStream_t)stream));
  return 0;
}

/* OUT[pos][n] = sum_k ACT[pos][k] W'[n][k] (+ bias[n]) on wgmma, fp32 accuracy (3xTF32); see include/hyena_b200.h */
HY_API size_t hyena_b200_proj_wimg_bytes(int N, int K) { return (N < 1 || K < 1) ? 0 : proj_wimg_bytes(N, K); }

HY_API int hyena_b200_proj_gemm(const float* act, int act_layout, const float* W, int ldw, int w_transposed,
                         const float* bias, const float* fir, float* out, int out_layout, int B, int L, int K, int N,
                         int l_begin, int l_len, void* wimg, size_t wimg_bytes, void* stream) {
  HY_CHECK(act && W && out && wimg, "null pointer");
  if (l_len <= 0) { l_begin = 0; l_len = L; }
  HY_CHECK(l_begin >= 0 && l_begin + l_len <= L, "position range [%d, %d) outside [0, %d)", l_begin, l_begin + l_len, L);
  HY_CHECK(B >= 1 && L >= 1 && K >= 1 && N >= 1, "bad shape B=%d L=%d K=%d N=%d", B, L, K, N);
  HY_CHECK((act_layout == 0 || act_layout == 1) && (out_layout == 0 || out_layout == 1), "bad layout code");
  HY_CHECK(!fir || act_layout == 1, "the fused transposed short filter needs a channel-major activation");
  HY_CHECK(aligned16(act) && aligned16(out) && aligned16(wimg) && (!bias || aligned16(bias)), "pointers must be 16-byte aligned");
  HY_CHECK(wimg_bytes >= proj_wimg_bytes(N, K), "weight image scratch too small: %zu < %zu", wimg_bytes, proj_wimg_bytes(N, K));
  HY_CHECK(ldw >= (w_transposed ? N : K), "ldw %d too small", ldw);
  HY_CUDA(launch_proj_gemm(act, act_layout, W, ldw, w_transposed, bias, fir, out, out_layout, B, L, K, N, l_begin, l_len,
                           reinterpret_cast<float*>(wimg), (cudaStream_t)stream));
  return 0;
}

HY_API size_t hyena_b200_proj_wgrad_scratch_bytes(int M, int N) { return (M < 1 || N < 1) ? 0 : proj_wgrad_scratch_bytes(M, N); }

HY_API int hyena_b200_proj_wgrad(const float* X, const float* Y, const float* fir, float* dW, int transposed_out, float beta,
                          int B, int L, int M, int N, void* scratch, size_t scratch_bytes, void* stream) {
  HY_CHECK(X && Y && dW && scratch, "null pointer");
  HY_CHECK(B >= 1 && L >= 1 && M >= 1 && N >= 1, "bad shape B=%d L=%d M=%d N=%d", B, L, M, N);
  HY_CHECK(aligned16(X) && aligned16(Y) && aligned16(scratch), "pointers must be 16-byte aligned");
  HY_CHECK(scratch_bytes >= proj_wgrad_scratch_bytes(M, N), "scratch too small: %zu < %zu", scratch_bytes,
           proj_wgrad_scratch_bytes(M, N));
  HY_CUDA(launch_proj_wgrad(X, Y, fir, dW, transposed_out, beta, B, L, M, N, reinterpret_cast<float*>(scratch),
                            (cudaStream_t)stream));
  return 0;
}

/* block MLP (fc1 -> gelu -> fc2) on the projection kernels with the GELU fused in; see include/hyena_b200.h */
static int check_gelu(int activation) {
  HY_CHECK(activation == HYENA_B200_GELU_TANH || activation == HYENA_B200_GELU_ERF,
           "activation %d: expected HYENA_B200_GELU_TANH (%d) or HYENA_B200_GELU_ERF (%d)", activation, HYENA_B200_GELU_TANH,
           HYENA_B200_GELU_ERF);
  return 0;
}

HY_API int hyena_b200_proj_gemm_gelu(const float* act, const float* W, int ldw, int w_transposed, const float* bias,
                                     int activation, float* out, int B, int L, int K, int N, void* wimg, size_t wimg_bytes,
                                     void* stream) {
  if (check_gelu(activation)) return 1;
  HY_CHECK(act && W && out && wimg, "null pointer");
  HY_CHECK(B >= 1 && L >= 1 && K >= 1 && N >= 1, "bad shape B=%d L=%d K=%d N=%d", B, L, K, N);
  HY_CHECK(aligned16(act) && aligned16(out) && aligned16(wimg) && (!bias || aligned16(bias)), "pointers must be 16-byte aligned");
  HY_CHECK(wimg_bytes >= proj_wimg_bytes(N, K), "weight image scratch too small: %zu < %zu", wimg_bytes, proj_wimg_bytes(N, K));
  HY_CHECK(ldw >= (w_transposed ? N : K), "ldw %d too small", ldw);
  HY_CUDA(launch_proj_gemm(act, 1, W, ldw, w_transposed, bias, nullptr, out, 1, B, L, K, N, 0, L, reinterpret_cast<float*>(wimg),
                           (cudaStream_t)stream, activation, nullptr));
  return 0;
}

HY_API int hyena_b200_proj_gemm_dgelu(const float* act, const float* W, int ldw, int w_transposed, const float* pre,
                                      int activation, float* out, int B, int L, int K, int N, void* wimg, size_t wimg_bytes,
                                      void* stream) {
  if (check_gelu(activation)) return 1;
  HY_CHECK(act && W && pre && out && wimg, "null pointer");
  HY_CHECK(B >= 1 && L >= 1 && K >= 1 && N >= 1, "bad shape B=%d L=%d K=%d N=%d", B, L, K, N);
  HY_CHECK(aligned16(act) && aligned16(out) && aligned16(wimg), "pointers must be 16-byte aligned");
  HY_CHECK(wimg_bytes >= proj_wimg_bytes(N, K), "weight image scratch too small: %zu < %zu", wimg_bytes, proj_wimg_bytes(N, K));
  HY_CHECK(ldw >= (w_transposed ? N : K), "ldw %d too small", ldw);
  const size_t n_out = (size_t)B * N * L;
  HY_CHECK(pre + n_out <= out || out + n_out <= pre, "pre and out must not overlap");
  HY_CUDA(launch_proj_gemm(act, 0, W, ldw, w_transposed, nullptr, nullptr, out, 0, B, L, K, N, 0, L, reinterpret_cast<float*>(wimg),
                           (cudaStream_t)stream, activation, pre));
  return 0;
}

HY_API int hyena_b200_proj_wgrad_gelu(const float* X, const float* Y, int activation, float* dW, int transposed_out, float beta,
                                      int B, int L, int M, int N, void* scratch, size_t scratch_bytes, void* stream) {
  if (check_gelu(activation)) return 1;
  HY_CHECK(X && Y && dW && scratch, "null pointer");
  HY_CHECK(B >= 1 && L >= 1 && M >= 1 && N >= 1, "bad shape B=%d L=%d M=%d N=%d", B, L, M, N);
  HY_CHECK(aligned16(X) && aligned16(Y) && aligned16(scratch), "pointers must be 16-byte aligned");
  HY_CHECK(scratch_bytes >= proj_wgrad_scratch_bytes(M, N), "scratch too small: %zu < %zu", scratch_bytes,
           proj_wgrad_scratch_bytes(M, N));
  HY_CUDA(launch_proj_wgrad(X, Y, nullptr, dW, transposed_out, beta, B, L, M, N, reinterpret_cast<float*>(scratch),
                            (cudaStream_t)stream, activation));
  return 0;
}

HY_API int hyena_b200_fftconv_fwd(const float* u, const float* kspec, const float* Dvec, float* out, int B, int H, int L,
                           void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(B, H, L)) return 1;
  HY_CHECK(u && kspec && Dvec && out, "null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, H, L, false, &c)) return 1;
  PassArgs a = base_args(B, H, L, T);
  a.A = c.A; a.kspec = reinterpret_cast<const float2*>(kspec);
  a.src = u; a.fbias = Dvec; a.out = out;
  a.vec = ((L & 1) == 0) && aligned8(u) && aligned8(out);
  for (int c0 = 0; c0 < H; c0 += c.nch) {
    const int n = (H - c0 < c.nch) ? H - c0 : c.nch;
    a.c0 = c0;
    HY_CUDA(launch_col_fwd(COL_PLAIN, a, n * B, s));
    HY_CUDA(launch_row_pass(ROW_CONV_FWD, a, n * B, s));
    HY_CUDA(launch_col_inv(INV_PLAIN_FWD, a, n * B, s));
  }
  return 0;
}

HY_API int hyena_b200_fftconv_fwd_windows(const float* u, const float* kspec, const float* Dvec, float* out,
                                          const long long* seg_base, const int* row_start, const int* out_start,
                                          long long total, int B, int H, int L, void* workspace, size_t workspace_bytes,
                                          void* stream) {
  if (check_windows(seg_base, row_start, out_start, total, B, H, L)) return 1;
  HY_CHECK(u && kspec && Dvec && out, "null pointer");
  HY_CHECK(aligned4(u) && aligned4(Dvec) && aligned4(out) && aligned8(kspec),
           "misaligned pointer: u, Dvec and out must be 4-byte aligned, kspec 8-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, H, L, false, &c)) return 1;
  PassArgs a = base_args(B, H, L, T);
  a.A = c.A; a.kspec = reinterpret_cast<const float2*>(kspec);
  a.src = u; a.fbias = Dvec; a.out = out;
  a.row_start = row_start; a.seg_base = seg_base; a.cstride = total; a.out_start = out_start;
  for (int c0 = 0; c0 < H; c0 += c.nch) {
    const int n = (H - c0 < c.nch) ? H - c0 : c.nch;
    a.c0 = c0;
    HY_CUDA(launch_col_fwd(COL_PLAIN_WIN, a, n * B, s));
    HY_CUDA(launch_row_pass(ROW_CONV_FWD, a, n * B, s));
    HY_CUDA(launch_col_inv(INV_PLAIN_FWD_WIN, a, n * B, s));
  }
  return 0;
}

HY_API int hyena_b200_fftconv_bwd(const float* dout, const float* u, const float* kspec, const float* Dvec, float* du,
                           float* dk, float* dD, int B, int H, int L, void* workspace, size_t workspace_bytes,
                           void* stream) {
  if (check_shape(B, H, L)) return 1;
  HY_CHECK(dout && u && kspec && Dvec && du && dk && dD, "null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, H, L, true, &c)) return 1;
  PassArgs a = base_args(B, H, L, T);
  a.kspec = reinterpret_cast<const float2*>(kspec);
  a.fbias = Dvec;
  a.vec = ((L & 1) == 0) && aligned8(u) && aligned8(dout) && aligned8(du) && aligned8(dk);
  for (int c0 = 0; c0 < H; c0 += c.nch) {
    const int n = (H - c0 < c.nch) ? H - c0 : c.nch;
    a.c0 = c0; a.B = B;
    a.A2 = c.A2; a.A3 = c.A3;
    a.A = c.A; a.src = dout;
    HY_CUDA(launch_col_fwd(COL_PLAIN, a, n * B, s));
    a.A = c.A2; a.src = u;
    HY_CUDA(launch_col_fwd(COL_PLAIN, a, n * B, s));
    a.A = c.A;
    HY_CUDA(launch_row_pass(ROW_CONV_BWD, a, n, s));
    a.src = u; a.src2 = dout; a.out = du; a.red = dD;
    HY_CUDA(launch_col_inv(INV_PLAIN_BWD, a, n * B, s));
    a.B = 1; a.out = dk;
    HY_CUDA(launch_col_inv(INV_DK, a, n, s));
  }
  return 0;
}

/* d deltas (D) = gradient of k = h * (exp(-t |deltas|) + shift) w.r.t. deltas (ExponentialModulation with modulation_lr != 0,
 * hyena.py:145-155); k is the filter the forward produced, dk its gradient, both (D, L); t (L). */
HY_API int hyena_b200_filter_ddelta(const float* dk, const float* k, const float* t, const float* deltas, float shift, int D,
                             int L, float* ddelta, void* stream) {
  HY_CHECK(D >= 1 && L >= 1 && dk && k && t && deltas && ddelta, "filter_ddelta: bad arguments");
  HY_CUDA(launch_filter_ddelta(dk, k, t, deltas, shift, D, L, ddelta, (cudaStream_t)stream));
  return 0;
}

/* normalized=True (hyena.py:235-236): out[c][t] = k[c][t] / norm[t], norm[t] = sum_c |k[c][t]|;  bwd: dk from dout, out, norm */
HY_API int hyena_b200_filter_l1norm_fwd(const float* k, float* out, float* norm, int D, int L, void* stream) {
  HY_CHECK(D >= 1 && L >= 1 && k && out && norm, "filter_l1norm_fwd: bad arguments");
  HY_CUDA(launch_l1norm_fwd(k, out, norm, D, L, (cudaStream_t)stream));
  return 0;
}
HY_API int hyena_b200_filter_l1norm_bwd(const float* dout, const float* out, const float* norm, float* dk, int D, int L,
                                 void* stream) {
  HY_CHECK(D >= 1 && L >= 1 && dout && out && norm && dk, "filter_l1norm_bwd: bad arguments");
  HY_CUDA(launch_l1norm_bwd(dout, out, norm, dk, D, L, (cudaStream_t)stream));
  return 0;
}

/* y = LayerNorm(x + res) * w + b, res_out = x + res (flash_attn/modules/block.py:111-148, pre-norm Block) */
HY_API size_t hyena_b200_add_layernorm_scratch_bytes(long long rows, int D) {
  return (rows < 1 || D < 1) ? 0 : (size_t)ln_partials(rows) * 2 * (size_t)D * sizeof(float);
}

HY_API int hyena_b200_add_layernorm_fwd(const float* x, const float* res, const float* w, const float* b, float eps,
                                 float* res_out, float* y, float* mean, float* rstd, long long rows, int D, void* stream) {
  HY_CHECK(rows >= 1 && D >= 1, "bad shape rows=%lld D=%d", rows, D);
  HY_CHECK(x && w && y && mean && rstd, "null pointer");
  HY_CHECK(res == nullptr || res_out != nullptr, "res_out is required when a residual is added");
  ln::FwdArgs a{x, res, w, b, res_out, y, mean, rstd, rows, D, eps};
  HY_CUDA(launch_add_ln_fwd(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_add_layernorm_bwd(const float* dy, const float* dres, const float* r, const float* w, const float* mean,
                                 const float* rstd, float* dx, float* dw, float* db, long long rows, int D, void* scratch,
                                 size_t scratch_bytes, void* stream) {
  HY_CHECK(rows >= 1 && D >= 1, "bad shape rows=%lld D=%d", rows, D);
  HY_CHECK(dy && r && w && mean && rstd && dx && dw && scratch, "null pointer");
  HY_CHECK(scratch_bytes >= hyena_b200_add_layernorm_scratch_bytes(rows, D), "scratch too small (%zu bytes)", scratch_bytes);
  ln::BwdArgs a{dy, dres, r, w, mean, rstd, dx, reinterpret_cast<float*>(scratch), rows, D};
  HY_CUDA(launch_add_ln_bwd(a, dw, db, (cudaStream_t)stream));
  return 0;
}

}  // extern "C"

// ---- incremental decoding: the checks and launches of every entry point, templates over the history element type
/* incremental decoding of the causal operator (the reference's HyenaOperator.recurrence hook, hyena.py:384-386) */
static int check_decode_shape(int B, int cache_B, int D, int order, int Lcap) {
  HY_CHECK(B >= 1 && D >= 1 && Lcap >= 1, "bad shape B=%d D=%d Lcap=%d", B, D, Lcap);
  HY_CHECK(B == cache_B, "batch size %d differs from the decode cache's %d", B, cache_B);
  HY_CHECK(order >= 2 && order <= dec::kMaxOrder, "order %d outside [2, %d]", order, dec::kMaxOrder);
  HY_CHECK(Lcap <= (1 << 20), "cache length %d exceeds the supported maximum %d", Lcap, 1 << 20);
  return 0;
}

template <class T>
static int decode_hist(const float* p, const float* in_bias, const float* sw, const float* sb, T* h, float* tail, int B,
                       int cache_B, int D, int order, int P, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail, "null pointer");
  HY_CHECK(P >= 1 && P <= Lcap, "prefill of %d positions outside [1, %d]", P, Lcap);
  dec::HistArgsT<T> a{p, in_bias, sw, sb, h, tail, B, D, (order + 1) * D, P, dec::ld_for(Lcap), (order - 1) * D,
                      nullptr};
  HY_CUDA(launch_decode_hist(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_hist_rows(const float* p, const float* in_bias, const float* sw, const float* sb, T* h, float* tail,
                            const int* row_start, int B, int cache_B, int D, int order, int P, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail && row_start, "null pointer");
  HY_CHECK(P >= 1 && P <= Lcap, "prefill of %d positions outside [1, %d]", P, Lcap);
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && elem_aligned(h) && aligned4(tail) && aligned4(row_start) &&
               (!in_bias || aligned4(in_bias)),
           "misaligned pointer: p, in_bias, sw, sb, h, tail and row_start must be 4-byte aligned");
  dec::HistArgsT<T> a{p, in_bias, sw, sb, h, tail, B, D, (order + 1) * D, P, dec::ld_for(Lcap), (order - 1) * D,
                      row_start};
  HY_CUDA(launch_decode_hist(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_admit(const float* p, const float* in_bias, const float* sw, const float* sb, T* h, float* tail,
                        const int* rows, const int* row_start, int k, int cache_B, int D, int order, int P, int t,
                        int Lcap, void* stream) {
  if (check_decode_shape(k, k, D, order, Lcap)) return 1;
  HY_CHECK(k <= cache_B, "%d prompts for a decode cache of %d rows", k, cache_B);
  HY_CHECK(p && sw && sb && h && tail && rows, "null pointer");
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && elem_aligned(h) && aligned4(tail) && aligned4(rows) &&
               (!in_bias || aligned4(in_bias)) && (!row_start || aligned4(row_start)),
           "misaligned pointer: p, in_bias, sw, sb, h, tail, rows and row_start must be 4-byte aligned");
  HY_CHECK(t >= 0 && t <= Lcap, "position %d outside the decode cache [0, %d]", t, Lcap);
  HY_CHECK(P >= 1 && P <= t, "a prompt of %d positions cannot end at position %d (it needs 1 <= P <= t)", P, t);
  dec::AdmitArgsT<T> a{{p, in_bias, sw, sb, h, tail, k, D, (order + 1) * D, P, dec::ld_for(Lcap), (order - 1) * D,
                        row_start}, rows, t - P, t};
  HY_CUDA(launch_decode_admit(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_admit_packed(const float* p, const float* in_bias, const float* sw, const float* sb, T* h, float* tail,
                               const int* rows, const long long* seg_base, const int* row_start, long long Tp, int k,
                               int cache_B, int D, int order, int P, int t, int Lcap, void* stream) {
  if (check_decode_shape(k, k, D, order, Lcap)) return 1;
  HY_CHECK(k <= cache_B, "%d prompts for a decode cache of %d rows", k, cache_B);
  HY_CHECK(p && sw && sb && h && tail && rows && seg_base && row_start, "null pointer");
  HY_CHECK(aligned4(p) && aligned4(sw) && aligned4(sb) && elem_aligned(h) && aligned4(tail) && aligned4(rows) &&
               aligned4(row_start) && aligned8(seg_base) && (!in_bias || aligned4(in_bias)),
           "misaligned pointer: p, in_bias, sw, sb, h, tail, rows and row_start must be 4-byte aligned, seg_base 8-byte");
  HY_CHECK(t >= 0 && t <= Lcap, "position %d outside the decode cache [0, %d]", t, Lcap);
  HY_CHECK(P >= 1 && P <= t, "a prompt of %d positions cannot end at position %d (it needs 1 <= P <= t)", P, t);
  HY_CHECK(Tp >= P, "bad packed length %lld: the channel stride must hold the longest prompt (%d)", Tp, P);
  dec::AdmitPackedArgsT<T> a{{{p, in_bias, sw, sb, h, tail, k, D, (order + 1) * D, P, dec::ld_for(Lcap), (order - 1) * D,
                               row_start}, rows, t - P, t}, seg_base, Tp};
  HY_CUDA(launch_decode_admit_packed(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_shift(T* h, int B, int D, int order, int t, int shift, int Lcap, void* stream) {
  if (check_decode_shape(B, B, D, order, Lcap)) return 1;
  HY_CHECK(h, "null pointer");
  HY_CHECK(hist_aligned(h), "%s", kAlignH<T>);
  HY_CHECK(t >= 0 && t <= Lcap, "position %d outside the decode cache [0, %d]", t, Lcap);
  HY_CHECK((shift & 3) == 0, "shift %d is not a multiple of 4", shift);
  HY_CHECK(shift >= -t, "left shift by %d past the start of a history of %d positions", -shift, t);
  HY_CHECK(shift <= Lcap - t, "right shift by %d moves position %d past the decode cache's %d", shift, t, Lcap);
  if (shift == 0) return 0;
  dec::ShiftArgsT<T> a{h, dec::ld_for(Lcap), t, shift};
  HY_CUDA(launch_decode_shift(a, (long long)(order - 1) * B * D, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_step(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                       const float* fbias, T* h, float* tail, float* s_t, const float* v_in, float* out, float* part,
                       int B, int cache_B, int D, int order, int o, int t, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(t >= 0 && t < Lcap, "position %d outside the decode cache [0, %d)", t, Lcap);
  const int ld = dec::ld_for(Lcap);
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  const int F = order - 1;
  dec::DotArgsT<T> dot{h, k + (size_t)o * ld, part, B, D, t, ld, F * ld, dec::chunks_for(Lcap)};
  dec::StepArgsT<T> st{part, (t + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o,
                       F * ld, F, ld, p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, t,
                       (order - 1 - o) * D, o == order - 2};
  HY_CUDA(launch_decode_step(dot, st, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_win_step(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                           const float* fbias, T* h, float* tail, float* s_t, const float* v_in, float* out,
                           float* part, const float* win, int B, int cache_B, int D, int order, int o, int t, int b,
                           int Wc, int W, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && win, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(b >= 0 && (b & 3) == 0, "window base %d must be a non-negative multiple of 4", b);
  HY_CHECK(Wc >= 1 && Wc <= W && b <= Lcap - Wc, "window [%d, %d) of width %d outside the decode cache [0, %d)", b,
           b + Wc, W, Lcap);
  HY_CHECK(t - b >= 0 && t - b < Wc, "position %d outside the window [%d, %d)", t, b, b + Wc);
  const int ld = dec::ld_for(Lcap);
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  const int F = order - 1;
  dec::DotArgsT<T> dot{h + b, k + (size_t)o * ld, part, B, D, t - b, ld, F * ld, dec::chunks_for(Lcap)};
  dec::WinStepArgsT<T> w{{part, (t - b + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(Lcap), k + (size_t)o * ld,
                          fbias + o, F * ld, F, ld, p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, B, D,
                          (order + 1) * D, order, t, (order - 1 - o) * D, o == order - 2}, win, W, t - b};
  HY_CUDA(launch_decode_win_step(dot, w, (cudaStream_t)stream));
  return 0;
}

/* extending a decode cache by n positions at once (decode_extend.cuh) */
static int check_extend_range(int t, int n, int Lcap) {
  HY_CHECK(n >= 1, "extend of %d positions: n must be >= 1", n);
  HY_CHECK(t >= 0 && t <= Lcap - n, "positions [%d, %d) outside the decode cache [0, %d)", t, t + n, Lcap);
  return 0;
}

HY_API int hyena_b200_decode_extend_groups(int B, int D, int t, int n) {
  if (B < 1 || D < 1 || t < 0 || n < 1) return 0;
  return dec::ext_groups(B, D, t, n);
}

template <class T>
static int decode_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb, T* h, float* tail,
                              float* s, int B, int cache_B, int D, int order, int t, int n, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail && s, "null pointer");
  dec::ExtHistArgsT<T> a{p, in_bias, sw, sb, tail, s, h, B, D, (order + 1) * D, t, n, dec::ld_for(Lcap),
                         (order - 1) * D};
  HY_CUDA(launch_decode_ext_hist(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_extend_dot(const T* h, const float* k, float* part, int groups, int B, int cache_B, int D, int order,
                             int o, int t, int n, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(h && k && part, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(groups == dec::ext_groups(B, D, t, n), "partials sized for %d groups; this extend needs %d "
           "(hyena_b200_decode_extend_groups)", groups, dec::ext_groups(B, D, t, n));
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  const int NT = dec::ext_tile(n);
  dec::ExtDotArgsT<T> a{h, k + (size_t)o * ld, part, B, D, t, n, ld, F * ld, (-t) & 3, (n + NT - 1) / NT,
                        dec::ext_chunks_per_cta(B, D, t, n), dec::chunks_for(t + n), groups};
  HY_CUDA(launch_decode_ext_dot(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_extend_combine(const float* part, long long row_stride, int j_stride, int groups, const float* fbias,
                                 const T* h, const float* s, void* out, int B, int cache_B, int D, int order, int o,
                                 int t, int n, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(part && fbias && h && s && out, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(groups >= 1 && j_stride >= 0 && row_stride >= 0, "bad partial layout: groups %d, strides %lld / %d", groups,
           row_stride, j_stride);
  if constexpr (!kFp32<T>)
    HY_CHECK(elem_aligned(h) && elem_aligned(static_cast<T*>(out)),
             "misaligned pointer: h and out must be 2-byte aligned");
  const int ld = dec::ld_for(Lcap), last = o == order - 2;
  dec::ExtCombineArgsT<T> a{part, row_stride, j_stride, groups, fbias + o, order - 1, h, s,
                            last ? nullptr : static_cast<T*>(out), last ? static_cast<float*>(out) : nullptr, B, D,
                            (order + 1) * D, t, n, ld, (order - 2 - o) * D, last};
  HY_CUDA(launch_decode_ext_combine(a, (cudaStream_t)stream));
  return 0;
}

/* decoding a branched cache (DecodeCache.fork): each of the R rows holds positions [b, b + Hc) of one branch with row
   stride H; the filter is the parent cache's (row stride ld = ld_for(Lcap)) and is addressed from k + ld - H
   (decode_args.h) */
static int check_branch(int R, int D, int order, int o, int t, int n, int b, int Hc, int H, int Lcap) {
  if (check_decode_shape(R, R, D, order, Lcap)) return 1;
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(b >= 0 && (b & 3) == 0, "branch base %d must be a non-negative multiple of 4", b);
  HY_CHECK(Hc >= 1 && b <= Lcap - Hc, "branch horizon [%d, %d) outside the decode cache [0, %d)", b, b + Hc, Lcap);
  HY_CHECK((H & 3) == 0 && H >= Hc && H <= dec::ld_for(Lcap) - b,
           "branch history width %d must be a multiple of 4 in [Hc, ld - b] = [%d, %d]", H, Hc, dec::ld_for(Lcap) - b);
  HY_CHECK(n >= 1 && t >= b && t <= b + Hc - n, "positions [%d, %d) outside the branch horizon [%d, %d)", t, t + n, b,
           b + Hc);
  return 0;
}

template <class T>
static int decode_branch_step(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                              const float* fbias, T* h, float* tail, float* s_t, const float* v_in, float* out,
                              float* part, const float* f, const int* parent, int R, int D, int order, int o, int t,
                              int b, int Hc, int H, int Lcap, void* stream) {
  if (check_branch(R, D, order, o, t, 1, b, Hc, H, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && f && parent, "null pointer");
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  const float* kb = k + (size_t)o * ld + (ld - H);
  dec::DotArgsT<T> dot{h, kb, part, R, D, t - b, H, F * ld, dec::chunks_for(H)};
  dec::BranchStepArgsT<T> w{{part, (t - b + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(H), kb, fbias + o, F * ld,
                             F, H, p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, R, D, (order + 1) * D, order, t - b,
                             (order - 1 - o) * D, o == order - 2}, f, parent};
  HY_CUDA(launch_decode_branch_step(dot, w, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_branch_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb, T* h,
                                     float* tail, float* s, int R, int D, int order, int t, int n, int b, int Hc, int H,
                                     int Lcap, void* stream) {
  if (check_branch(R, D, order, 0, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail && s, "null pointer");
  dec::ExtHistArgsT<T> a{p, in_bias, sw, sb, tail, s, h, R, D, (order + 1) * D, t - b, n, H, (order - 1) * D};
  HY_CUDA(launch_decode_ext_hist(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_branch_extend_dot(const T* h, const float* k, float* part, int groups, int R, int D, int order, int o,
                                    int t, int n, int b, int Hc, int H, int Lcap, void* stream) {
  if (check_branch(R, D, order, o, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(h && k && part, "null pointer");
  HY_CHECK(groups == dec::ext_groups(R, D, t - b, n), "partials sized for %d groups; this extend needs %d "
           "(hyena_b200_decode_extend_groups with t - b)", groups, dec::ext_groups(R, D, t - b, n));
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  const int ld = dec::ld_for(Lcap), F = order - 1, NT = dec::ext_tile(n), j = t - b;
  dec::ExtDotArgsT<T> a{h, k + (size_t)o * ld + (ld - H), part, R, D, j, n, H, F * ld, (-j) & 3, (n + NT - 1) / NT,
                        dec::ext_chunks_per_cta(R, D, j, n), dec::chunks_for(j + n), groups};
  HY_CUDA(launch_decode_ext_dot(a, (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_branch_combine(const float* part, long long row_stride, int j_stride, int groups, const float* fbias,
                                 const T* h, const float* s, void* out, const float* f, const int* parent, int R, int D,
                                 int order, int o, int t, int n, int b, int Hc, int H, int Lcap, void* stream) {
  if (check_branch(R, D, order, o, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(part && fbias && h && s && out && f && parent, "null pointer");
  HY_CHECK(groups >= 1 && j_stride >= 0 && row_stride >= 0, "bad partial layout: groups %d, strides %lld / %d", groups,
           row_stride, j_stride);
  if constexpr (!kFp32<T>)
    HY_CHECK(elem_aligned(h) && elem_aligned(static_cast<T*>(out)),
             "misaligned pointer: h and out must be 2-byte aligned");
  const int last = o == order - 2;
  dec::BranchCombineArgsT<T> a{{part, row_stride, j_stride, groups, fbias + o, order - 1, h, s,
                                last ? nullptr : static_cast<T*>(out), last ? static_cast<float*>(out) : nullptr, R, D,
                                (order + 1) * D, t - b, n, H, (order - 2 - o) * D, last}, f, parent};
  HY_CUDA(launch_decode_branch_combine(a, (cudaStream_t)stream));
  return 0;
}

/* device-position steps (a step captured once in a CUDA graph): the kernels read pos = [t, win_b, base] */
template <class T>
static int check_dev_step(int o, int order, const float* p_t, const float* sw, const float* sb, const float* tail,
                          const float* v_in, const float* k, const T* h, const int* pos) {
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(pos && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "null or misaligned device position");
  HY_CHECK(aligned16(k) && hist_aligned(h), "%s", kAlignKH<T>);
  return 0;
}

template <class T>
static int decode_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                           const float* fbias, T* h, float* tail, float* s_t, const float* v_in, float* out,
                           float* part, const int* pos, int B, int cache_B, int D, int order, int o, int t_max,
                           int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  HY_CHECK(t_max >= 1 && t_max <= Lcap, "position bound %d outside [1, %d]", t_max, Lcap);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  dec::DotArgsT<T> dot{h, k + (size_t)o * ld, part, B, D, 0, ld, F * ld, dec::chunks_for(Lcap)};
  dec::StepArgsT<T> st{part, 0, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o, F * ld, F, ld, p_t, in_bias, sw,
                       sb, tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, 0, (order - 1 - o) * D,
                       o == order - 2};
  HY_CUDA(launch_decode_step_dev(dot, st, pos, dec::chunks_for(t_max), (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_win_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                               const float* fbias, T* h, float* tail, float* s_t, const float* v_in, float* out,
                               float* part, const float* win, const int* pos, int B, int cache_B, int D, int order,
                               int o, int W, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && win, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  HY_CHECK(W >= 1 && W <= Lcap, "window width %d outside [1, %d]", W, Lcap);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  dec::DotArgsT<T> dot{h, k + (size_t)o * ld, part, B, D, 0, ld, F * ld, dec::chunks_for(Lcap)};
  dec::WinStepArgsT<T> w{{part, 0, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o, F * ld, F, ld, p_t, in_bias,
                          sw, sb, tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, 0, (order - 1 - o) * D,
                          o == order - 2}, win, W, 0};
  HY_CUDA(launch_decode_win_step_dev(dot, w, pos, dec::chunks_for(W), (cudaStream_t)stream));
  return 0;
}

template <class T>
static int decode_branch_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                  const float* k, const float* fbias, T* h, float* tail, float* s_t, const float* v_in,
                                  float* out, float* part, const float* f, const int* parent, const int* pos, int R,
                                  int D, int order, int o, int H, int Lcap, void* stream) {
  if (check_decode_shape(R, R, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && f && parent, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  const int ld = dec::ld_for(Lcap), F = order - 1;
  HY_CHECK((H & 3) == 0 && H >= 4 && H <= ld, "branch history width %d must be a multiple of 4 in [4, %d]", H, ld);
  const float* kb = k + (size_t)o * ld + (ld - H);
  dec::DotArgsT<T> dot{h, kb, part, R, D, 0, H, F * ld, dec::chunks_for(H)};
  dec::BranchStepArgsT<T> w{{part, 0, dec::chunks_for(H), kb, fbias + o, F * ld, F, H, p_t, in_bias, sw, sb, tail, s_t,
                             v_in, h, out, R, D, (order + 1) * D, order, 0, (order - 1 - o) * D, o == order - 2}, f,
                            parent};
  HY_CUDA(launch_decode_branch_step_dev(dot, w, pos, dec::chunks_for(H), (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_pos_advance(int* pos, void* stream) {
  HY_CHECK(pos && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "null or misaligned device position");
  HY_CUDA(launch_decode_pos_advance(pos, (cudaStream_t)stream));
  return 0;
}

/* ---- the C entry points of the decoding kernels: fp32 history (hyena_b200_decode_*) and 16-bit history
   (hyena_b200_decode_*_h16, the same arguments after a history dtype code; include/hyena_b200.h) */
template <class F>
static int with_hist_type(int hist_dtype, F&& f) {
  if (hist_dtype == HYENA_B200_HIST_F16) return f(__half());
  if (hist_dtype == HYENA_B200_HIST_BF16) return f(__nv_bfloat16());
  return fail("unknown history dtype code %d (%d: fp16, %d: bf16; an fp32 history uses the entry points without _h16)",
              hist_dtype, HYENA_B200_HIST_F16, HYENA_B200_HIST_BF16);
}

extern "C" {

HY_API int hyena_b200_decode_hist(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                  float* tail, int B, int cache_B, int D, int order, int P, int Lcap, void* stream) {
  return decode_hist<float>(p, in_bias, sw, sb, h, tail, B, cache_B, D, order, P, Lcap, stream);
}
HY_API int hyena_b200_decode_hist_h16(int hist_dtype, const float* p, const float* in_bias, const float* sw,
                                      const float* sb, void* h, float* tail, int B, int cache_B, int D, int order,
                                      int P, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_hist<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, B, cache_B, D, order, P, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_hist_rows(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                       float* tail, const int* row_start, int B, int cache_B, int D, int order, int P,
                                       int Lcap, void* stream) {
  return decode_hist_rows<float>(p, in_bias, sw, sb, h, tail, row_start, B, cache_B, D, order, P, Lcap, stream);
}
HY_API int hyena_b200_decode_hist_rows_h16(int hist_dtype, const float* p, const float* in_bias, const float* sw,
                                           const float* sb, void* h, float* tail, const int* row_start, int B,
                                           int cache_B, int D, int order, int P, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_hist_rows<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, row_start, B, cache_B, D, order, P, Lcap,
                               stream);
  });
}

HY_API int hyena_b200_decode_admit(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                   float* tail, const int* rows, const int* row_start, int k, int cache_B, int D,
                                   int order, int P, int t, int Lcap, void* stream) {
  return decode_admit<float>(p, in_bias, sw, sb, h, tail, rows, row_start, k, cache_B, D, order, P, t, Lcap, stream);
}
HY_API int hyena_b200_decode_admit_h16(int hist_dtype, const float* p, const float* in_bias, const float* sw,
                                       const float* sb, void* h, float* tail, const int* rows, const int* row_start,
                                       int k, int cache_B, int D, int order, int P, int t, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_admit<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, rows, row_start, k, cache_B, D, order, P, t,
                           Lcap, stream);
  });
}

HY_API int hyena_b200_decode_admit_packed(const float* p, const float* in_bias, const float* sw, const float* sb,
                                          float* h, float* tail, const int* rows, const long long* seg_base,
                                          const int* row_start, long long Tp, int k, int cache_B, int D, int order, int P,
                                          int t, int Lcap, void* stream) {
  return decode_admit_packed<float>(p, in_bias, sw, sb, h, tail, rows, seg_base, row_start, Tp, k, cache_B, D, order, P, t,
                                    Lcap, stream);
}
HY_API int hyena_b200_decode_admit_packed_h16(int hist_dtype, const float* p, const float* in_bias, const float* sw,
                                              const float* sb, void* h, float* tail, const int* rows,
                                              const long long* seg_base, const int* row_start, long long Tp, int k,
                                              int cache_B, int D, int order, int P, int t, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_admit_packed<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, rows, seg_base, row_start, Tp, k, cache_B,
                                  D, order, P, t, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_shift(float* h, int B, int D, int order, int t, int shift, int Lcap, void* stream) {
  return decode_shift<float>(h, B, D, order, t, shift, Lcap, stream);
}
HY_API int hyena_b200_decode_shift_h16(int hist_dtype, void* h, int B, int D, int order, int t, int shift, int Lcap,
                                       void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_shift<T>(static_cast<T*>(h), B, D, order, t, shift, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                  const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                  const float* v_in, float* out, float* part, int B, int cache_B, int D, int order,
                                  int o, int t, int Lcap, void* stream) {
  return decode_step<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, B, cache_B, D, order, o, t,
                            Lcap, stream);
}
HY_API int hyena_b200_decode_step_h16(int hist_dtype, const float* p_t, const float* in_bias, const float* sw,
                                      const float* sb, const float* k, const float* fbias, void* h, float* tail,
                                      float* s_t, const float* v_in, float* out, float* part, int B, int cache_B, int D,
                                      int order, int o, int t, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_step<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, B, cache_B, D,
                          order, o, t, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_win_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const float* win, int B, int cache_B,
                                      int D, int order, int o, int t, int b, int Wc, int W, int Lcap, void* stream) {
  return decode_win_step<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, win, B, cache_B, D,
                                order, o, t, b, Wc, W, Lcap, stream);
}
HY_API int hyena_b200_decode_win_step_h16(int hist_dtype, const float* p_t, const float* in_bias, const float* sw,
                                          const float* sb, const float* k, const float* fbias, void* h, float* tail,
                                          float* s_t, const float* v_in, float* out, float* part, const float* win,
                                          int B, int cache_B, int D, int order, int o, int t, int b, int Wc, int W,
                                          int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_win_step<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, win, B,
                              cache_B, D, order, o, t, b, Wc, W, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb,
                                         float* h, float* tail, float* s, int B, int cache_B, int D, int order, int t,
                                         int n, int Lcap, void* stream) {
  return decode_extend_hist<float>(p, in_bias, sw, sb, h, tail, s, B, cache_B, D, order, t, n, Lcap, stream);
}
HY_API int hyena_b200_decode_extend_hist_h16(int hist_dtype, const float* p, const float* in_bias, const float* sw,
                                             const float* sb, void* h, float* tail, float* s, int B, int cache_B, int D,
                                             int order, int t, int n, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_extend_hist<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, s, B, cache_B, D, order, t, n, Lcap,
                                 stream);
  });
}

HY_API int hyena_b200_decode_extend_dot(const float* h, const float* k, float* part, int groups, int B, int cache_B,
                                        int D, int order, int o, int t, int n, int Lcap, void* stream) {
  return decode_extend_dot<float>(h, k, part, groups, B, cache_B, D, order, o, t, n, Lcap, stream);
}
HY_API int hyena_b200_decode_extend_dot_h16(int hist_dtype, const void* h, const float* k, float* part, int groups,
                                            int B, int cache_B, int D, int order, int o, int t, int n, int Lcap,
                                            void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_extend_dot<T>(static_cast<const T*>(h), k, part, groups, B, cache_B, D, order, o, t, n, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_extend_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out, int B,
                                            int cache_B, int D, int order, int o, int t, int n, int Lcap,
                                            void* stream) {
  return decode_extend_combine<float>(part, row_stride, j_stride, groups, fbias, h, s, out, B, cache_B, D, order, o, t,
                                      n, Lcap, stream);
}
HY_API int hyena_b200_decode_extend_combine_h16(int hist_dtype, const float* part, long long row_stride, int j_stride,
                                                int groups, const float* fbias, const void* h, const float* s,
                                                void* out, int B, int cache_B, int D, int order, int o, int t, int n,
                                                int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_extend_combine<T>(part, row_stride, j_stride, groups, fbias, static_cast<const T*>(h), s, out, B,
                                    cache_B, D, order, o, t, n, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_branch_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                         const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                         const float* v_in, float* out, float* part, const float* f, const int* parent,
                                         int R, int D, int order, int o, int t, int b, int Hc, int H, int Lcap,
                                         void* stream) {
  return decode_branch_step<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, f, parent, R, D,
                                   order, o, t, b, Hc, H, Lcap, stream);
}
HY_API int hyena_b200_decode_branch_step_h16(int hist_dtype, const float* p_t, const float* in_bias, const float* sw,
                                             const float* sb, const float* k, const float* fbias, void* h, float* tail,
                                             float* s_t, const float* v_in, float* out, float* part, const float* f,
                                             const int* parent, int R, int D, int order, int o, int t, int b, int Hc,
                                             int H, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_branch_step<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, f,
                                 parent, R, D, order, o, t, b, Hc, H, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_branch_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb,
                                                float* h, float* tail, float* s, int R, int D, int order, int t, int n,
                                                int b, int Hc, int H, int Lcap, void* stream) {
  return decode_branch_extend_hist<float>(p, in_bias, sw, sb, h, tail, s, R, D, order, t, n, b, Hc, H, Lcap, stream);
}
HY_API int hyena_b200_decode_branch_extend_hist_h16(int hist_dtype, const float* p, const float* in_bias,
                                                    const float* sw, const float* sb, void* h, float* tail, float* s,
                                                    int R, int D, int order, int t, int n, int b, int Hc, int H,
                                                    int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_branch_extend_hist<T>(p, in_bias, sw, sb, static_cast<T*>(h), tail, s, R, D, order, t, n, b, Hc, H,
                                        Lcap, stream);
  });
}

HY_API int hyena_b200_decode_branch_extend_dot(const float* h, const float* k, float* part, int groups, int R, int D,
                                               int order, int o, int t, int n, int b, int Hc, int H, int Lcap,
                                               void* stream) {
  return decode_branch_extend_dot<float>(h, k, part, groups, R, D, order, o, t, n, b, Hc, H, Lcap, stream);
}
HY_API int hyena_b200_decode_branch_extend_dot_h16(int hist_dtype, const void* h, const float* k, float* part,
                                                   int groups, int R, int D, int order, int o, int t, int n, int b,
                                                   int Hc, int H, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_branch_extend_dot<T>(static_cast<const T*>(h), k, part, groups, R, D, order, o, t, n, b, Hc, H, Lcap,
                                       stream);
  });
}

HY_API int hyena_b200_decode_branch_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out,
                                            const float* f, const int* parent, int R, int D, int order, int o, int t,
                                            int n, int b, int Hc, int H, int Lcap, void* stream) {
  return decode_branch_combine<float>(part, row_stride, j_stride, groups, fbias, h, s, out, f, parent, R, D, order, o,
                                      t, n, b, Hc, H, Lcap, stream);
}
HY_API int hyena_b200_decode_branch_combine_h16(int hist_dtype, const float* part, long long row_stride, int j_stride,
                                                int groups, const float* fbias, const void* h, const float* s,
                                                void* out, const float* f, const int* parent, int R, int D, int order,
                                                int o, int t, int n, int b, int Hc, int H, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_branch_combine<T>(part, row_stride, j_stride, groups, fbias, static_cast<const T*>(h), s, out, f,
                                    parent, R, D, order, o, t, n, b, Hc, H, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const int* pos, int B, int cache_B,
                                      int D, int order, int o, int t_max, int Lcap, void* stream) {
  return decode_step_dev<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, pos, B, cache_B, D,
                                order, o, t_max, Lcap, stream);
}
HY_API int hyena_b200_decode_step_dev_h16(int hist_dtype, const float* p_t, const float* in_bias, const float* sw,
                                          const float* sb, const float* k, const float* fbias, void* h, float* tail,
                                          float* s_t, const float* v_in, float* out, float* part, const int* pos, int B,
                                          int cache_B, int D, int order, int o, int t_max, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_step_dev<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, pos, B,
                              cache_B, D, order, o, t_max, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_win_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                          const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                          const float* v_in, float* out, float* part, const float* win, const int* pos,
                                          int B, int cache_B, int D, int order, int o, int W, int Lcap, void* stream) {
  return decode_win_step_dev<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, win, pos, B, cache_B,
                                    D, order, o, W, Lcap, stream);
}
HY_API int hyena_b200_decode_win_step_dev_h16(int hist_dtype, const float* p_t, const float* in_bias, const float* sw,
                                              const float* sb, const float* k, const float* fbias, void* h, float* tail,
                                              float* s_t, const float* v_in, float* out, float* part, const float* win,
                                              const int* pos, int B, int cache_B, int D, int order, int o, int W,
                                              int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_win_step_dev<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, win,
                                  pos, B, cache_B, D, order, o, W, Lcap, stream);
  });
}

HY_API int hyena_b200_decode_branch_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                             const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                             const float* v_in, float* out, float* part, const float* f,
                                             const int* parent, const int* pos, int R, int D, int order, int o, int H,
                                             int Lcap, void* stream) {
  return decode_branch_step_dev<float>(p_t, in_bias, sw, sb, k, fbias, h, tail, s_t, v_in, out, part, f, parent, pos, R,
                                       D, order, o, H, Lcap, stream);
}
HY_API int hyena_b200_decode_branch_step_dev_h16(int hist_dtype, const float* p_t, const float* in_bias,
                                                 const float* sw, const float* sb, const float* k, const float* fbias,
                                                 void* h, float* tail, float* s_t, const float* v_in, float* out,
                                                 float* part, const float* f, const int* parent, const int* pos, int R,
                                                 int D, int order, int o, int H, int Lcap, void* stream) {
  return with_hist_type(hist_dtype, [&](auto tag) { using T = decltype(tag);
    return decode_branch_step_dev<T>(p_t, in_bias, sw, sb, k, fbias, static_cast<T*>(h), tail, s_t, v_in, out, part, f,
                                     parent, pos, R, D, order, o, H, Lcap, stream);
  });
}

}  // extern "C"
