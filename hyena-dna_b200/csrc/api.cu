// C ABI of libhyena_b200.so (include/hyena_b200.h): argument checks, workspace carving, row-group
// scheduling of the three FFT passes.  No torch types; PyTorch hands in raw device pointers.
#include <atomic>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

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
static thread_local bool g_prof_suppress = false;   // inside a pipelined call: the kernels of different row groups overlap, so
                                                    // the call is timed as ONE record on the caller's stream instead

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
  if (!g_prof_on || g_prof_suppress || capturing(s)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_cur_e0 = get_event();
  cudaEventRecord(g_cur_e0, s);
}
void prof_end(int kind, cudaStream_t s) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (!g_prof_on || !g_cur_e0 || g_prof_suppress) return;
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

static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

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

// ---------------------------------------------------------------- pipelined row groups (L2-resident scratch)
// The three passes of a row group are enqueued back to back on one of S auxiliary streams, group g on stream g % S with
// scratch slot g % S, G channels per group: the inter-pass scratch of a group (G x B x 8 MB at M = 2^20) is re-read while
// it is still in the 50 MB L2, a slot is overwritten in place by the next group of its stream (dirty lines never
// have to reach DRAM), and kernels of different groups overlap so that the short launches leave no idle tails.
// In-stream order carries every dependency (passes of a group, reuse of a slot); the caller's stream forks into the
// auxiliary streams and joins them again, so to the caller the call is ordered on its own stream as before.
// HYENA_B200_PIPE="S,G" (0 = off: one launch per pass over all rows).
struct PipeCfg { int S, G; };
static PipeCfg pipe_cfg() {
  static PipeCfg c = [] {
    PipeCfg v{0, 0};
    const char* e = getenv("HYENA_B200_PIPE");
    int s = 0, g = 0;
    if (e && sscanf(e, "%d,%d", &s, &g) == 2 && s >= 1 && s <= 8 && g >= 1) { v.S = s; v.G = g; }
    return v;
  }();
  return c;
}
struct PipeDev { cudaStream_t st[8]; cudaEvent_t fork; cudaEvent_t join[8]; int n = 0; std::mutex mu; };
static PipeDev g_pipe[64];
static int get_pipe(int S, PipeDev** out) {
  int dev = -1;
  HY_CUDA(cudaGetDevice(&dev));
  HY_CHECK(dev >= 0 && dev < 64, "unsupported device ordinal %d", dev);
  std::lock_guard<std::mutex> lk(g_mu);
  PipeDev& p = g_pipe[dev];
  if (p.n == 0) HY_CUDA(cudaEventCreateWithFlags(&p.fork, cudaEventDisableTiming));
  while (p.n < S) {
    HY_CUDA(cudaStreamCreateWithFlags(&p.st[p.n], cudaStreamNonBlocking));
    HY_CUDA(cudaEventCreateWithFlags(&p.join[p.n], cudaEventDisableTiming));
    ++p.n;
  }
  *out = &p;
  return 0;
}
// RAII: fork the caller's stream into S auxiliary streams; join() makes the caller's stream wait for all of them
struct PipeRun {
  PipeDev* p = nullptr; int S = 0; cudaStream_t main = nullptr; int kind = -1; bool active = false;
  std::unique_lock<std::mutex> lk;
  int begin(int S_, cudaStream_t main_, int kind_) {
    S = S_; main = main_; kind = kind_;
    if (get_pipe(S, &p)) return 1;
    lk = std::unique_lock<std::mutex>(p->mu);
    prof_begin(kind, main);
    g_prof_suppress = true;
    HY_CUDA(cudaEventRecord(p->fork, main));
    for (int i = 0; i < S; ++i) HY_CUDA(cudaStreamWaitEvent(p->st[i], p->fork, 0));
    active = true;
    return 0;
  }
  cudaStream_t stream(int g) const { return p->st[g % S]; }
  int join() {
    for (int i = 0; i < S; ++i) {
      HY_CUDA(cudaEventRecord(p->join[i], p->st[i]));
      HY_CUDA(cudaStreamWaitEvent(main, p->join[i], 0));
    }
    g_prof_suppress = false;
    active = false;
    prof_end(kind, main);
    g_launches.fetch_sub(1, std::memory_order_relaxed);     // the span record is not a kernel launch
    return 0;
  }
  ~PipeRun() { if (active) { g_prof_suppress = false; for (int i = 0; i < S; ++i) { cudaEventRecord(p->join[i], p->st[i]); cudaStreamWaitEvent(main, p->join[i], 0); } } }
};

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
      "filter_fwd", "filter_bwd", "short_conv_bwd", "twiddle_init", "filter_tc_prep", "filter_tc_fwd", "filter_tc_bwd", "filter_tc_red", "fused_conv_fwd",
      "spectrum_convert", "proj_prep", "proj_gemm", "proj_wgrad",
      "conv_fwd<pipelined>", "conv_bwd<pipelined>", "filter_spectrum<pipelined>", "add_layer_norm", "filter_extra",
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
  const PipeCfg pc = pipe_cfg();
  if (pc.S > 0) {                                   // S scratch slots of G channels each
    const int g = pc.G < D ? pc.G : D;
    return hyena_b200_workspace_min_bytes(B, D, L, backward) * (size_t)g * (size_t)pc.S;
  }
  int nch = channels_per_group(group_budget_bytes(), B, D, L);
  if (nch < 1) nch = 1;
  return hyena_b200_workspace_min_bytes(B, D, L, backward) * (size_t)nch;
}

// tensor-core filter path: scratch for the tf32 hi/lo weight images (~0.3 MB, grow-only), one per (device, stream): two
// operators driven from different streams never share it (the prep kernel of one would overwrite the images the other's
// wgmma kernel is still reading)
static int get_wimg(int D, cudaStream_t stream, float** out) {
  int dev = -1;
  HY_CUDA(cudaGetDevice(&dev));
  HY_CHECK(dev >= 0 && dev < 64, "unsupported device ordinal %d", dev);
  std::lock_guard<std::mutex> lk(g_mu);
  struct Buf { float* p = nullptr; size_t n = 0; };
  static std::map<std::pair<int, cudaStream_t>, Buf> bufs;
  Buf& b = bufs[std::make_pair(dev, stream)];
  const size_t need = filter_tc_wimg_bytes(D);
  if (b.n < need) {
    if (b.p) { HY_CUDA(cudaStreamSynchronize(stream)); HY_CUDA(cudaFree(b.p)); b.p = nullptr; b.n = 0; }
    HY_CUDA(cudaMalloc(&b.p, need));
    b.n = need;
  }
  *out = b.p;
  return 0;
}

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
  static const bool simt = getenv("HYENA_B200_FILTER") && !strcmp(getenv("HYENA_B200_FILTER"), "simt");
  if (simt) {
    HY_CUDA(launch_filter_fwd(P, k_out, (cudaStream_t)stream));
    return 0;
  }
  float* wimg = nullptr;
  if (get_wimg(D, (cudaStream_t)stream, &wimg)) return 1;
  HY_CUDA(launch_filter_fwd_tc(P, wimg, k_out, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_filter_bwd(const float* z, int z_stride, const float* t, const float* W0, const float* b0,
                          const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                          const float* freq, const float* deltas, float shift, int modulate, int L, int E, int N,
                          int D, const float* dk, float* dW0, float* db0, float* dW1, float* db1, float* dW2,
                          float* db2, float* dW3, float* dfreq, float* dz, int dz_stride, void* stream) {
  FilterParams P;
  if (fill_filter_params(&P, z, z_stride, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, E, N, D))
    return 1;
  HY_CHECK(dk && dW0 && db0 && dW1 && db1 && dW2 && db2 && dW3 && dfreq, "null gradient pointer");
  FilterGrads G{dW0, db0, dW1, db1, dW2, db2, dW3, dfreq, dz, dz_stride};
  HY_CUDA(launch_filter_bwd(P, dk, G, (cudaStream_t)stream));
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
  RedLaunch r{dh, scratch, zT, dW0, db0, dW1, db1, dW2, db2, dW3, dfreq, L, D, E};
  HY_CUDA(launch_filter_red_tc(r, (cudaStream_t)stream));
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
  const PipeCfg pc = pipe_cfg();
  const int G = pc.G < D ? pc.G : D;
  if (pc.S > 0 && c.nch >= G * pc.S && D > G) {
    PipeRun run;
    if (run.begin(pc.S, s, K_PIPE_FILTER)) return 1;
    const size_t slot = (row_bytes(L) / sizeof(float2)) * (size_t)G;
    int g = 0;
    for (int c0 = 0; c0 < D; c0 += G, ++g) {
      const int n = (D - c0 < G) ? D - c0 : G;
      a.c0 = c0; a.A = c.A + slot * (size_t)(g % pc.S);
      HY_CUDA(launch_col_fwd(COL_FILTER, a, n, run.stream(g)));
      HY_CUDA(launch_row_pass(ROW_FILTER, a, n, run.stream(g)));
    }
    return run.join();
  }
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

HY_API int hyena_b200_core_fwd(const float* p, const float* in_bias, const float* sw, const float* sb, const float* kspec,
                        const float* fbias, float* y_pre, float* c_save, float* gspec_save, int B, int D, int L,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (check_shape(B, D, L)) return 1;
  HY_CHECK(p && sw && sb && kspec && fbias && y_pre, "null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, D, L, false, &c)) return 1;
  PassArgs a = base_args(B, D, L, T);
  a.A = c.A; a.kspec = reinterpret_cast<const float2*>(kspec);
  a.p = p; a.in_bias = in_bias; a.sw = sw; a.sb = sb; a.fbias = fbias; a.out = y_pre; a.out2 = c_save;
  a.gspec = reinterpret_cast<float2*>(gspec_save);
  a.vec = ((L & 1) == 0) && aligned8(p) && aligned8(y_pre) && (!c_save || aligned8(c_save));
  a.stage = ((L & 3) == 0) && aligned16(p) && !getenv("HYENA_B200_NO_STAGE");
  const PipeCfg pc = pipe_cfg();
  const int G = pc.G < D ? pc.G : D;
  if (pc.S > 0 && c.nch >= G * pc.S && D > G) {
    PipeRun run;
    if (run.begin(pc.S, s, K_PIPE_FWD)) return 1;
    const size_t slot = (row_bytes(L) / sizeof(float2)) * (size_t)B * (size_t)G;
    int g = 0;
    for (int c0 = 0; c0 < D; c0 += G, ++g) {
      const int n = (D - c0 < G) ? D - c0 : G;
      cudaStream_t st = run.stream(g);
      a.c0 = c0; a.A = c.A + slot * (size_t)(g % pc.S);
      HY_CUDA(launch_col_fwd(COL_GATE, a, n * B, st));
      HY_CUDA(launch_row_pass(ROW_CONV_FWD, a, n * B, st));
      HY_CUDA(launch_col_inv(INV_CONV_FWD, a, n * B, st));
    }
    return run.join();
  }
  for (int c0 = 0; c0 < D; c0 += c.nch) {
    const int n = (D - c0 < c.nch) ? D - c0 : c.nch;
    a.c0 = c0;
    HY_CUDA(launch_col_fwd(COL_GATE, a, n * B, s));
    HY_CUDA(launch_row_pass(ROW_CONV_FWD, a, n * B, s));
    HY_CUDA(launch_col_inv(INV_CONV_FWD, a, n * B, s));
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
  cudaStream_t s = (cudaStream_t)stream;
  Twiddles T;
  if (get_twiddles(s, &T)) return 1;
  Carve c;
  if (carve(workspace, workspace_bytes, B, D, L, true, &c)) return 1;
  PassArgs a = base_args(B, D, L, T);
  a.kspec = reinterpret_cast<const float2*>(kspec);
  a.p = p; a.in_bias = in_bias; a.sw = sw; a.sb = sb; a.fbias = fbias;
  a.vec = ((L & 1) == 0) && aligned8(p) && aligned8(dy_pre) && aligned8(c_saved) && aligned8(dk) &&
          aligned8(ds_scratch);
  a.stage = ((L & 3) == 0) && aligned16(p) && aligned16(dy_pre) && aligned16(c_saved) && !getenv("HYENA_B200_NO_STAGE");
  const PipeCfg pc = pipe_cfg();
  const int G = pc.G < D ? pc.G : D;
  const bool piped = pc.S > 0 && c.nch >= G * pc.S && D > G;
  PipeRun run;
  if (piped && run.begin(pc.S, s, K_PIPE_BWD)) return 1;
  const int step = piped ? G : c.nch;
  const size_t rowE = row_bytes(L) / sizeof(float2);
  int g = 0;
  for (int c0 = 0; c0 < D; c0 += step, ++g) {
    const int n = (D - c0 < step) ? D - c0 : step;
    if (piped) {                                  // slot g % S: [A: G*B rows][A2: G*B rows][A3: G rows]
      s = run.stream(g);
      c.A = reinterpret_cast<float2*>(workspace) + rowE * (size_t)(2 * B + 1) * (size_t)G * (size_t)(g % pc.S);
      c.A2 = c.A + rowE * (size_t)B * (size_t)G;
      c.A3 = c.A2 + rowE * (size_t)B * (size_t)G;
    }
    a.c0 = c0; a.B = B;
    a.A2 = c.A2; a.A3 = c.A3;
    a.A = c.A; a.src = dy_pre;
    HY_CUDA(launch_col_fwd(COL_DC, a, n * B, s));        // A  <- columns of dc = dy_pre * x0
    a.gspec = const_cast<float2*>(reinterpret_cast<const float2*>(gspec_saved));
    if (!gspec_saved) {
      a.A = c.A2;
      HY_CUDA(launch_col_fwd(COL_GATE, a, n * B, s));    // A2 <- columns of g = v * x1 (recomputed)
    }
    a.A = c.A;
    static const bool bwd1 = !(getenv("HYENA_B200_ROW_BWD1") && !strcmp(getenv("HYENA_B200_ROW_BWD1"), "0"));
    // (the 128-thread batch-1 kernel exists for 1024-point rows only)
    HY_CUDA(launch_row_pass((B == 1 && gspec_saved && bwd1 && a.logM2 == 10) ? ROW_CONV_BWD1 : ROW_CONV_BWD, a, n, s));   // A <- rows of dg, A3 <- rows of dk
    a.src = dy_pre; a.src2 = c_saved; a.out2 = ds_scratch; a.red = dfbias; a.dsw = dsw; a.dsb = dsb;
    HY_CUDA(launch_col_inv(INV_BWD_DG, a, n * B, s));
    a.B = 1; a.out = dk;
    HY_CUDA(launch_col_inv(INV_DK, a, n, s));
  }
  if (piped) { if (run.join()) return 1; s = (cudaStream_t)stream; }
  // pass 3 already accumulated dsw / dsb from the operand windows it had staged: no second read of p here.
  // dp == NULL: the caller consumes ds directly (hyena_b200_proj_gemm / proj_wgrad apply the transposed short filter on
  // the fly and d in_proj.bias follows from dsb and two edge samples), so dp never exists in HBM.
  if (dp) {
    ShortBwdArgs sa{ds_scratch, nullptr, in_bias, sw, dp, dsw, dsb, d_in_bias, L, 3 * D, a.vec && aligned8(dp)};
    HY_CUDA(launch_short_bwd(sa, B, s));
  }
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

/* incremental decoding of the causal operator (the reference's HyenaOperator.recurrence hook, hyena.py:384-386) */
static int check_decode_shape(int B, int cache_B, int D, int order, int Lcap) {
  HY_CHECK(B >= 1 && D >= 1 && Lcap >= 1, "bad shape B=%d D=%d Lcap=%d", B, D, Lcap);
  HY_CHECK(B == cache_B, "batch size %d differs from the decode cache's %d", B, cache_B);
  HY_CHECK(order >= 2 && order <= dec::kMaxOrder, "order %d outside [2, %d]", order, dec::kMaxOrder);
  HY_CHECK(Lcap <= (1 << 20), "cache length %d exceeds the supported maximum %d", Lcap, 1 << 20);
  return 0;
}

HY_API int hyena_b200_decode_hist(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                  float* tail, int B, int cache_B, int D, int order, int P, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail, "null pointer");
  HY_CHECK(P >= 1 && P <= Lcap, "prefill of %d positions outside [1, %d]", P, Lcap);
  dec::HistArgs a{p, in_bias, sw, sb, h, tail, B, D, (order + 1) * D, P, dec::ld_for(Lcap), (order - 1) * D};
  HY_CUDA(launch_decode_hist(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_step(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                                  const float* fbias, float* h, float* tail, float* s_t, const float* v_in, float* out,
                                  float* part, int B, int cache_B, int D, int order, int o, int t, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(t >= 0 && t < Lcap, "position %d outside the decode cache [0, %d)", t, Lcap);
  const int ld = dec::ld_for(Lcap);
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  const int F = order - 1;
  dec::DotArgs dot{h, k + (size_t)o * ld, part, B, D, t, ld, F * ld, dec::chunks_for(Lcap)};
  dec::StepArgs st{part, (t + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o, F * ld, F,
                   ld, p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, t, (order - 1 - o) * D,
                   o == order - 2};
  HY_CUDA(launch_decode_step(dot, st, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_win_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const float* win, int B, int cache_B,
                                      int D, int order, int o, int t, int b, int Wc, int W, int Lcap, void* stream) {
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
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  const int F = order - 1;
  dec::DotArgs dot{h + b, k + (size_t)o * ld, part, B, D, t - b, ld, F * ld, dec::chunks_for(Lcap)};
  dec::WinStepArgs w{{part, (t - b + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o,
                      F * ld, F, ld, p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, t,
                      (order - 1 - o) * D, o == order - 2},
                     win, W, t - b};
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

HY_API int hyena_b200_decode_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                         float* tail, float* s, int B, int cache_B, int D, int order, int t, int n, int Lcap,
                                         void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail && s, "null pointer");
  dec::ExtHistArgs a{p, in_bias, sw, sb, tail, s, h, B, D, (order + 1) * D, t, n, dec::ld_for(Lcap), (order - 1) * D};
  HY_CUDA(launch_decode_ext_hist(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_extend_dot(const float* h, const float* k, float* part, int groups, int B, int cache_B, int D,
                                        int order, int o, int t, int n, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(h && k && part, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(groups == dec::ext_groups(B, D, t, n), "partials sized for %d groups; this extend needs %d "
           "(hyena_b200_decode_extend_groups)", groups, dec::ext_groups(B, D, t, n));
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  const int ld = dec::ld_for(Lcap), F = order - 1;
  const int NT = dec::ext_tile(n);
  dec::ExtDotArgs a{h, k + (size_t)o * ld, part, B, D, t, n, ld, F * ld, (-t) & 3, (n + NT - 1) / NT,
                    dec::ext_chunks_per_cta(B, D, t, n), dec::chunks_for(t + n), groups};
  HY_CUDA(launch_decode_ext_dot(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_extend_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out, int B,
                                            int cache_B, int D, int order, int o, int t, int n, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap) || check_extend_range(t, n, Lcap)) return 1;
  HY_CHECK(part && fbias && h && s && out, "null pointer");
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(groups >= 1 && j_stride >= 0 && row_stride >= 0, "bad partial layout: groups %d, strides %lld / %d", groups,
           row_stride, j_stride);
  const int ld = dec::ld_for(Lcap), last = o == order - 2;
  dec::ExtCombineArgs a{part, row_stride, j_stride, groups, fbias + o, order - 1, h, s, last ? nullptr : out,
                        last ? out : nullptr, B, D, (order + 1) * D, t, n, ld, (order - 2 - o) * D, last};
  HY_CUDA(launch_decode_ext_combine(a, (cudaStream_t)stream));
  return 0;
}

/* decoding a branched cache (DecodeCache.fork): each of the R rows holds positions [b, b + Hc) of one branch with row stride
   H; the filter is the parent cache's (row stride ld = ld_for(Lcap)) and is addressed from k + ld - H (decode_args.h) */
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

HY_API int hyena_b200_decode_branch_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                         const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                         const float* v_in, float* out, float* part, const float* f, const int* parent,
                                         int R, int D, int order, int o, int t, int b, int Hc, int H, int Lcap,
                                         void* stream) {
  if (check_branch(R, D, order, o, t, 1, b, Hc, H, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && f && parent, "null pointer");
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  const int ld = dec::ld_for(Lcap), F = order - 1;
  const float* kb = k + (size_t)o * ld + (ld - H);
  dec::DotArgs dot{h, kb, part, R, D, t - b, H, F * ld, dec::chunks_for(H)};
  dec::BranchStepArgs w{{part, (t - b + dec::kChunk - 1) / dec::kChunk, dec::chunks_for(H), kb, fbias + o, F * ld, F, H,
                         p_t, in_bias, sw, sb, tail, s_t, v_in, h, out, R, D, (order + 1) * D, order, t - b,
                         (order - 1 - o) * D, o == order - 2},
                        f, parent};
  HY_CUDA(launch_decode_branch_step(dot, w, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_branch_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb,
                                                float* h, float* tail, float* s, int R, int D, int order, int t, int n,
                                                int b, int Hc, int H, int Lcap, void* stream) {
  if (check_branch(R, D, order, 0, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(p && sw && sb && h && tail && s, "null pointer");
  dec::ExtHistArgs a{p, in_bias, sw, sb, tail, s, h, R, D, (order + 1) * D, t - b, n, H, (order - 1) * D};
  HY_CUDA(launch_decode_ext_hist(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_branch_extend_dot(const float* h, const float* k, float* part, int groups, int R, int D,
                                               int order, int o, int t, int n, int b, int Hc, int H, int Lcap,
                                               void* stream) {
  if (check_branch(R, D, order, o, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(h && k && part, "null pointer");
  HY_CHECK(groups == dec::ext_groups(R, D, t - b, n), "partials sized for %d groups; this extend needs %d "
           "(hyena_b200_decode_extend_groups with t - b)", groups, dec::ext_groups(R, D, t - b, n));
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  const int ld = dec::ld_for(Lcap), F = order - 1, NT = dec::ext_tile(n), j = t - b;
  dec::ExtDotArgs a{h, k + (size_t)o * ld + (ld - H), part, R, D, j, n, H, F * ld, (-j) & 3, (n + NT - 1) / NT,
                    dec::ext_chunks_per_cta(R, D, j, n), dec::chunks_for(j + n), groups};
  HY_CUDA(launch_decode_ext_dot(a, (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_branch_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out,
                                            const float* f, const int* parent, int R, int D, int order, int o, int t,
                                            int n, int b, int Hc, int H, int Lcap, void* stream) {
  if (check_branch(R, D, order, o, t, n, b, Hc, H, Lcap)) return 1;
  HY_CHECK(part && fbias && h && s && out && f && parent, "null pointer");
  HY_CHECK(groups >= 1 && j_stride >= 0 && row_stride >= 0, "bad partial layout: groups %d, strides %lld / %d", groups,
           row_stride, j_stride);
  const int last = o == order - 2;
  dec::BranchCombineArgs a{{part, row_stride, j_stride, groups, fbias + o, order - 1, h, s, last ? nullptr : out,
                            last ? out : nullptr, R, D, (order + 1) * D, t - b, n, H, (order - 2 - o) * D, last},
                           f, parent};
  HY_CUDA(launch_decode_branch_combine(a, (cudaStream_t)stream));
  return 0;
}

/* device-position steps (a step captured once in a CUDA graph): the kernels read pos = [t, win_b, base] */
static int check_dev_step(int o, int order, const float* p_t, const float* sw, const float* sb, const float* tail,
                          const float* v_in, const float* k, const float* h, const int* pos) {
  HY_CHECK(o >= 0 && o < order - 1, "recurrence %d outside [0, %d)", o, order - 1);
  HY_CHECK(o == 0 ? (p_t && sw && sb && tail && !v_in) : (v_in != nullptr),
           o == 0 ? "null pointer: recurrence 0 needs p_t, sw, sb, tail (and no v_in)" : "null pointer: v_in");
  HY_CHECK(pos && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "null or misaligned device position");
  HY_CHECK(aligned16(k) && aligned16(h), "k and h must be 16-byte aligned");
  return 0;
}

HY_API int hyena_b200_decode_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const int* pos, int B, int cache_B, int D,
                                      int order, int o, int t_max, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  HY_CHECK(t_max >= 1 && t_max <= Lcap, "position bound %d outside [1, %d]", t_max, Lcap);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  dec::DotArgs dot{h, k + (size_t)o * ld, part, B, D, 0, ld, F * ld, dec::chunks_for(Lcap)};
  dec::StepArgs st{part, 0, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o, F * ld, F, ld, p_t, in_bias, sw, sb, tail,
                   s_t, v_in, h, out, B, D, (order + 1) * D, order, 0, (order - 1 - o) * D, o == order - 2};
  HY_CUDA(launch_decode_step_dev(dot, st, pos, dec::chunks_for(t_max), (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_win_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                          const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                          const float* v_in, float* out, float* part, const float* win, const int* pos, int B,
                                          int cache_B, int D, int order, int o, int W, int Lcap, void* stream) {
  if (check_decode_shape(B, cache_B, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && win, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  HY_CHECK(W >= 1 && W <= Lcap, "window width %d outside [1, %d]", W, Lcap);
  const int ld = dec::ld_for(Lcap), F = order - 1;
  dec::DotArgs dot{h, k + (size_t)o * ld, part, B, D, 0, ld, F * ld, dec::chunks_for(Lcap)};
  dec::WinStepArgs w{{part, 0, dec::chunks_for(Lcap), k + (size_t)o * ld, fbias + o, F * ld, F, ld, p_t, in_bias, sw, sb,
                      tail, s_t, v_in, h, out, B, D, (order + 1) * D, order, 0, (order - 1 - o) * D, o == order - 2},
                     win, W, 0};
  HY_CUDA(launch_decode_win_step_dev(dot, w, pos, dec::chunks_for(W), (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_branch_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                             const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                             const float* v_in, float* out, float* part, const float* f, const int* parent,
                                             const int* pos, int R, int D, int order, int o, int H, int Lcap, void* stream) {
  if (check_decode_shape(R, R, D, order, Lcap)) return 1;
  HY_CHECK(k && fbias && h && s_t && out && part && f && parent, "null pointer");
  if (check_dev_step(o, order, p_t, sw, sb, tail, v_in, k, h, pos)) return 1;
  const int ld = dec::ld_for(Lcap), F = order - 1;
  HY_CHECK((H & 3) == 0 && H >= 4 && H <= ld, "branch history width %d must be a multiple of 4 in [4, %d]", H, ld);
  const float* kb = k + (size_t)o * ld + (ld - H);
  dec::DotArgs dot{h, kb, part, R, D, 0, H, F * ld, dec::chunks_for(H)};
  dec::BranchStepArgs w{{part, 0, dec::chunks_for(H), kb, fbias + o, F * ld, F, H, p_t, in_bias, sw, sb, tail, s_t, v_in, h,
                         out, R, D, (order + 1) * D, order, 0, (order - 1 - o) * D, o == order - 2},
                        f, parent};
  HY_CUDA(launch_decode_branch_step_dev(dot, w, pos, dec::chunks_for(H), (cudaStream_t)stream));
  return 0;
}

HY_API int hyena_b200_decode_pos_advance(int* pos, void* stream) {
  HY_CHECK(pos && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "null or misaligned device position");
  HY_CUDA(launch_decode_pos_advance(pos, (cudaStream_t)stream));
  return 0;
}

}  // extern "C"
