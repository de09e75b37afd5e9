/* hyena_b200 -- C ABI of the sm_90a Hyena long-convolution library (libhyena_b200.so).
 *
 * This is the drop-in boundary for the HyenaOperator hot path of HazyResearch/hyena-dna.  The
 * reference's own FFI for this path is the pybind11 module `fftconv`
 * (csrc/fftconv/fftconv.cpp:238-241: fftconv_fwd / fftconv_bwd) called from
 * src/ops/fftconv.py:58-108, plus the PyTorch graph of src/models/sequence/hyena.py:388-444.
 * Every entry point below names the reference interface it replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers (fp32, contiguous, 8-byte aligned unless stated); sizes are
 *     element counts; `stream` is a cudaStream_t passed as void*.
 *   - inputs are borrowed and never written; outputs are fully overwritten unless marked (+=).
 *   - every function returns 0 on success and a non-zero code on failure; the message of the last
 *     failure on the calling thread is returned by hyena_b200_last_error().  Nothing here falls
 *     back to a CPU path: without a CUDA device the calls fail.
 *   - the functions are stateless and re-entrant apart from a per-device table of FFT twiddles that
 *     is built on first use; they enqueue work on `stream` and return without synchronising.
 *   - sequence length limit: L <= hyena_b200_max_seqlen() (= 2^20).  The reference extension stops at
 *     L <= 8192 (csrc/fftconv/fftconv.cpp:114-115).
 *
 * Layouts (B batch, D channels = d_model, L positions, N = filter_order = 64, E = emb_dim)
 *   p      (B, 3D, L)  in_proj output, channel-major, WITHOUT in_proj.bias (passed separately);
 *                      channels [0,D) = x0, [D,2D) = x1, [2D,3D) = v   (hyena.py:404)
 *   k      (D, L)      time-domain filter, channel-major
 *   kspec  (D, M) complex64 (interleaved re,im), M = hyena_b200_spectrum_elems(L): packed half-size
 *                      spectrum of k in the library's internal [k1][k2] order -- opaque to callers
 *   y_pre  (B, D, L)   operator output before out_proj, channel-major (hyena.py:432 before the rearrange)
 */
#ifndef HYENA_B200_H
#define HYENA_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: hyena_b200_proj_debug_buffer removed (the wgmma projection kernels keep no per-role counters) */
#define HYENA_B200_ABI_VERSION 2
#if defined(__GNUC__)
#define HY_API __attribute__((visibility("default")))
#else
#define HY_API
#endif

HY_API int hyena_b200_abi_version(void);
HY_API const char* hyena_b200_last_error(void);
/* number of CUDA kernels this library has launched since it was loaded (all threads) */
HY_API unsigned long long hyena_b200_launch_count(void);
HY_API int hyena_b200_max_seqlen(void);

/* Optional per-launch timing with CUDA events on the launching stream (used by bench.py's roofline leg).
 * profile_begin() starts a window; profile_end() synchronises the device and returns, per kernel class
 * (index < hyena_b200_kind_count(), name from hyena_b200_kind_name), the summed device milliseconds and the launch count. */
HY_API int hyena_b200_profile_begin(void);
HY_API int hyena_b200_profile_end(double* ms_by_kind, unsigned long long* launches_by_kind, int n);
HY_API const char* hyena_b200_kind_name(int kind);
HY_API int hyena_b200_kind_count(void);

/* M: complex elements per channel of a filter spectrum for sequence length L (power of two >= L, >= 1024) */
HY_API size_t hyena_b200_spectrum_elems(int L);
/* scratch bytes the conv entry points want for (B, D, L); backward != 0 for the *_bwd calls.
 * Any size >= hyena_b200_workspace_min_bytes() works; more lets more rows be in flight per launch. */
HY_API size_t hyena_b200_workspace_bytes(int B, int D, int L, int backward);
HY_API size_t hyena_b200_workspace_min_bytes(int B, int D, int L, int backward);

/* ---- implicit filter -------------------------------------------------------------------------
 * replaces HyenaFilter.filter (src/models/sequence/hyena.py:229-238): PositionalEmbedding rows
 * z (L,E; row stride z_stride) and t (L), Sin-MLP (hyena.py:96-106, :199-215), ExponentialModulation
 * (hyena.py:152-155).  Output k (D, L) channel-major == filter(L)[0].transpose(0,1).
 * N (filter_order) must be 64; E odd in [3,15]. */
HY_API int hyena_b200_filter_fwd(const float* z, int z_stride, const float* t,
                          const float* W0, const float* b0, const float* W1, const float* b1,
                          const float* W2, const float* b2, const float* W3,
                          const float* freq, const float* deltas, float shift, int modulate,
                          int L, int E, int N, int D, float* k_out, void* stream);

/* autograd of the above (the reference relies on torch autograd; closed form restated in DESIGN.md).
 * dk (D,L) -> parameter grads, all (+=) so callers zero them; dz (L,E; row stride dz_stride) may be NULL. */
HY_API int hyena_b200_filter_bwd(const float* z, int z_stride, const float* t,
                          const float* W0, const float* b0, const float* W1, const float* b1,
                          const float* W2, const float* b2, const float* W3,
                          const float* freq, const float* deltas, float shift, int modulate,
                          int L, int E, int N, int D, const float* dk,
                          float* dW0, float* db0, float* dW1, float* db1, float* dW2, float* db2,
                          float* dW3, float* dfreq, float* dz, int dz_stride, void* stream);

/* Tensor-core (wgmma, 3xTF32) backward in two stages.  Stage 1: per position, recompute the activations and back-
 * propagate through the MLP, writing dh = dk * modulation (D,L) and seven feature-major (64,L) arrays into `scratch`
 * (7*64*L floats, 16-byte aligned): a1, a2, a3, dp1, dp2, dp3, X.  Stage 2: the parameter gradients are reductions
 * over the sequence, done as accumulating wgmma GEMMs with K = position (all outputs (+=); zT is z transposed,
 * (E,L)); D <= 256, E <= 8:
 *   dW3 = dh a3^T, dW2 = dp3 a2^T, dW1 = dp2 a1^T, dW0 = dp1 z, db_l = rowsum(dp_{l+1}), dfreq = rowsum(X) */
HY_API int hyena_b200_filter_bwd_stage1(const float* z, int z_stride, const float* t,
                                 const float* W0, const float* b0, const float* W1, const float* b1,
                                 const float* W2, const float* b2, const float* W3,
                                 const float* freq, const float* deltas, float shift, int modulate,
                                 int L, int E, int N, int D, const float* dk, float* dh, float* scratch, void* stream);

HY_API int hyena_b200_filter_bwd_stage2(const float* dh, const float* scratch, const float* zT,
                                 float* dW0, float* db0, float* dW1, float* db1, float* dW2, float* db2,
                                 float* dW3, float* dfreq, int L, int E, int D, void* stream);

/* ---- filter spectrum -------------------------------------------------------------------------
 * replaces `k_f = torch.fft.rfft(k, n=fft_size) / fft_size` (hyena.py:62, src/ops/fftconv.py:65). */
HY_API int hyena_b200_filter_spectrum(const float* k, float* kspec, int D, int L,
                               void* workspace, size_t workspace_bytes, void* stream);

/* ---- fused operator core ---------------------------------------------------------------------
 * replaces hyena.py:394-432 for order=2: short_filter (depthwise Conv1d k=3, :363-369,:394), split
 * (:404), gate v*x1 (:420), fftconv_ref with bias skip term (:59-88 via :261), gate *x0 (:432).
 *   sw (3D,3) = short_filter.weight[:,0,:], sb (3D) = short_filter.bias, in_bias (3D) = in_proj.bias
 *   or NULL, fbias (D) = filter_fn.bias.  c_save (B,D,L) receives the fftconv output (needed by
 *   core_bwd) when non-NULL.  gspec_save ((D*B) rows of M complex64, row = c*B + b; may be NULL) receives the
 *   packed spectrum of the gated input g = short(v)*short(x1); handing it back to core_bwd saves one column
 *   pass and one row FFT per (b,c) row there (the reference saves u_f the same way, hyena.py:41). */
HY_API int hyena_b200_core_fwd(const float* p, const float* in_bias, const float* sw, const float* sb,
                        const float* kspec, const float* fbias,
                        float* y_pre, float* c_save, float* gspec_save, int B, int D, int L,
                        void* workspace, size_t workspace_bytes, void* stream);

/* backward of core_fwd (closed form: hyena.py:43-56 FFTConvFuncv2.backward,
 * csrc/fftconv/fftconv_cuda.cu:1157-1179).  dy_pre (B,D,L).  Outputs: dp (B,3D,L), dk (D,L);
 * (+=): dsw (3D,3), dsb (3D), dfbias (D), d_in_bias (3D, may be NULL).
 * ds_scratch (B,3D,L) receives ds, the gradient w.r.t. the short-filter OUTPUTS.  With dp == NULL the transposed short
 * filter pass is skipped (d_in_bias is then not written): hand ds to hyena_b200_proj_gemm / hyena_b200_proj_wgrad with
 * fir = sw, which apply dp[t] = w2 ds[t] + w1 ds[t+1] + w0 ds[t+2] in registers. */
HY_API int hyena_b200_core_bwd(const float* dy_pre, const float* p, const float* in_bias, const float* sw,
                        const float* sb, const float* kspec, const float* fbias, const float* c_saved,
                        const float* gspec_saved /* from core_fwd, or NULL to recompute */,
                        float* dp, float* dk, float* dsw, float* dsb, float* dfbias, float* d_in_bias,
                        float* ds_scratch, int B, int D, int L,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- plain long convolution (the reference extension's own surface) ---------------------------
 * fftconv_fwd replaces csrc/fftconv/fftconv.cpp:53-132 for fp32, gelu=false, no dropout mask, no q/v,
 * head_dim=1:  out[b,h,:] = causal_conv(u[b,h,:], k[h,:]) + u[b,h,:] * Dvec[h]     (fftconv_ref,
 * src/ops/fftconv.py:15-34).  The filter is passed as the opaque kspec from hyena_b200_filter_spectrum.
 * fftconv_bwd replaces fftconv.cpp:134-236 + src/ops/fftconv.py:87-103: du (B,H,L), dk (H,L) time
 * domain (the reference returns dk_f and inverts it in Python), dD (H) (+=). */
HY_API int hyena_b200_fftconv_fwd(const float* u, const float* kspec, const float* Dvec, float* out,
                           int B, int H, int L, void* workspace, size_t workspace_bytes, void* stream);
HY_API int hyena_b200_fftconv_bwd(const float* dout, const float* u, const float* kspec, const float* Dvec,
                           float* du, float* dk, float* dD, int B, int H, int L,
                           void* workspace, size_t workspace_bytes, void* stream);

/* ---- the reference extension's filter convention ---------------------------------------------
 * csrc/fftconv/fftconv.cpp:53-61 takes `filter = torch.fft.rfft(k, n=fft_size)`: (H, fft_size/2+1) complex64, natural
 * bin order, unnormalised (src/ops/fftconv.py:64-65); fftconv.cpp:134-143,235 returns `dfilter` in the same layout with
 * irfft(dfilter, n=fft_size, norm='forward')[:L] == dk (src/ops/fftconv.py:94-98).  These two entry points convert
 * between that convention and the packed kspec / the time-domain dk of fftconv_fwd / fftconv_bwd above, so that an
 * unmodified src/ops/fftconv.py:FFTConvFunc binds to this library (INTEGRATION.md).  fft_size: power of two >= 16 with
 * L <= fft_size/2 (fftconv.cpp:114-115).  k_scratch (H*L floats) is needed only when fft_size < 2*spectrum_elems(L);
 * kspec_scratch (H * spectrum_elems(L) complex64) only when fft_size == 2*spectrum_elems(L). */
HY_API int hyena_b200_spectrum_from_rfft(const float* filter, int fft_size, float* kspec, float* k_scratch, int H, int L,
                                  void* workspace, size_t workspace_bytes, void* stream);
HY_API int hyena_b200_spectrum_to_rfft(const float* dk, int fft_size, float* dfilter, float* kspec_scratch, int H, int L,
                                void* workspace, size_t workspace_bytes, void* stream);

/* ---- projections (library GEMM at the boundary of the custom-kernel span) ------------------------
 * in_proj / out_proj (hyena.py:350-351, :391, :440) are plain GEMMs and stay cuBLASLt calls.  These two
 * entry points run them on the CUDA 12.9 cuBLASLt with CUBLAS_COMPUTE_32F_EMULATED_16BFX9 (fp32 emulated
 * on bf16 tensor cores, fp32-level accuracy).  Column-major, strided-batched:
 * C[m,n] = alpha * op(A) op(B) + beta * C (+ bias[m]); op: 0 = N, 1 = T. */
HY_API int hyena_b200_gemm_available(void);

/* ---- projections on this library's own tensor-core kernel (csrc/proj_gemm.cuh) --------------------
 * The same GEMMs as above without the library call: wgmma, fp32 accuracy through 3xTF32, weights streamed by
 * TMA bulk copies, the activation converted on the fly into wgmma register fragments.  Computes, for every batch b,
 *     OUT[pos][n] = sum_k ACT[pos][k] * Wl[n][k] (+ bias[n]),    Wl[n][k] = w_transposed ? W[k*ldw + n] : W[n*ldw + k]
 *   act_layout 0: ACT is (B, L, K) row-major (u, dy: hyena.py:391, :440 backward)
 *              1: ACT is (B, K, L) channel-major (y_pre, ds: hyena.py:432-440)
 *   out_layout 0: OUT is (B, N, L) channel-major (p, dy_pre);   1: OUT is (B, L, N) row-major (y, du)
 *   fir (K,3) non-NULL (act_layout 1 only): ACT is ds, the gradient w.r.t. the short-filter OUTPUT, and the GEMM consumes
 *              dp[k][t] = fir[k][2] ds[k][t] + fir[k][1] ds[k][t+1] + fir[k][0] ds[k][t+2] (backward of the depthwise
 *              Conv1d, hyena.py:363-369) computed in registers -- dp never exists in HBM.
 *   l_begin, l_len: only positions [l_begin, l_begin + l_len) of every batch are computed (host-side pipelining of a
 *              long sequence against PCIe copies, hyena-dna_b200/host.py); l_len <= 0 means all L positions.
 *   wimg: scratch of hyena_b200_proj_wimg_bytes(N, K) bytes (tf32 hi/lo images of the weights, rebuilt every call). */
/* Weight gradients of the projections (hyena.py:391, :440 backward), reduction over the sequence positions:
 *     dW[m][n] (= or +=) sum_{b,pos} X[b][m][pos] * Y[b][pos][n]
 * X (B, M, L) channel-major (ds / y_pre), Y (B, L, N) row-major (u / dy); split-K over the SMs with the accumulators in
 * tensor memory, deterministic reduction of the partials.  transposed_out: dW is stored (N, M).  beta: 0 overwrite, else
 * dW = beta * dW + sum.  fir (M,3): X is ds and the transposed short filter is applied on the fly (see proj_gemm).
 * scratch: hyena_b200_proj_wgrad_scratch_bytes(M, N) bytes. */
HY_API size_t hyena_b200_proj_wgrad_scratch_bytes(int M, int N);
HY_API int hyena_b200_proj_wgrad(const float* X, const float* Y, const float* fir, float* dW, int transposed_out, float beta,
                          int B, int L, int M, int N, void* scratch, size_t scratch_bytes, void* stream);
HY_API size_t hyena_b200_proj_wimg_bytes(int N, int K);
HY_API int hyena_b200_proj_gemm(const float* act, int act_layout, const float* W, int ldw, int w_transposed,
                         const float* bias, const float* fir, float* out, int out_layout, int B, int L, int K, int N,
                         int l_begin, int l_len, void* wimg, size_t wimg_bytes, void* stream);
/* ---- block MLP: fc1 -> gelu -> fc2 with the GELU fused into the projection kernels ------------------
 * replaces flash_attn/modules/mlp.py:26-30 (Mlp.forward: fc1, activation, fc2) as src/models/sequence/long_conv_lm.py:102-123
 * (create_mlp_cls) builds it, and its autograd.  The hidden activation a = fc1(x) is kept channel-major (B, H, L): fc1
 * and its gradients are plain hyena_b200_proj_gemm / hyena_b200_proj_wgrad calls, and the three products of fc2 below apply
 * the activation (or its derivative) in registers, so gelu(a) and gelu'(a) never exist in HBM.  activation:
 * HYENA_B200_GELU_TANH = F.gelu(approximate="tanh"), HYENA_B200_GELU_ERF = F.gelu(approximate="none"), fp32 as torch
 * computes them.  Shapes, weights (W, ldw, w_transposed), wimg and scratch as for proj_gemm / proj_wgrad.
 *   proj_gemm_gelu   OUT (B, L, N) = gelu(ACT) Wl^T (+ bias),  ACT (B, K, L) channel-major        (fc2 forward)
 *   proj_gemm_dgelu  OUT (B, N, L) = (ACT Wl^T)^T o gelu'(pre), ACT (B, L, K) row-major, pre (B, N, L) the
 *                    pre-activation, not overlapping OUT                                          (fc2 input gradient)
 *   proj_wgrad_gelu  dW[m][n] (= or +=) sum_{b,pos} gelu(X[b][m][pos]) Y[b][pos][n]               (fc2 weight gradient) */
#define HYENA_B200_GELU_TANH 1
#define HYENA_B200_GELU_ERF 2
HY_API int hyena_b200_proj_gemm_gelu(const float* act, const float* W, int ldw, int w_transposed, const float* bias,
                                     int activation, float* out, int B, int L, int K, int N, void* wimg, size_t wimg_bytes,
                                     void* stream);
HY_API int hyena_b200_proj_gemm_dgelu(const float* act, const float* W, int ldw, int w_transposed, const float* pre,
                                      int activation, float* out, int B, int L, int K, int N, void* wimg, size_t wimg_bytes,
                                      void* stream);
HY_API int hyena_b200_proj_wgrad_gelu(const float* X, const float* Y, int activation, float* dW, int transposed_out, float beta,
                                      int B, int L, int M, int N, void* scratch, size_t scratch_bytes, void* stream);
HY_API int hyena_b200_gemm(int transa, int transb, int m, int n, int k, float alpha, const float* A, int lda,
                           long long strideA, const float* B, int ldb, long long strideB, float beta, float* C,
                           int ldc, long long strideC, int batch, const float* bias, int emulate, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- filter options outside the shipped configs -------------------------------------------------
 * modulation_lr != 0 (hyena.py:145-150: deltas is a Parameter): d deltas (D) from the filter k (D, L) the forward produced and
 * its gradient dk (D, L); t (L) = PositionalEmbedding.t.  Overwrites ddelta. */
HY_API int hyena_b200_filter_ddelta(const float* dk, const float* k, const float* t, const float* deltas, float shift, int D,
                             int L, float* ddelta, void* stream);
/* normalized=True (hyena.py:235-236, L1 norm over the channel dim of (1, L, D)): out[c][t] = k[c][t] / norm[t],
 * norm[t] = sum_c |k[c][t]| (L values, kept for the backward); bwd: dk = (dout - sign(out) * sum_c dout*out) / norm. */
HY_API int hyena_b200_filter_l1norm_fwd(const float* k, float* out, float* norm, int D, int L, void* stream);
HY_API int hyena_b200_filter_l1norm_bwd(const float* dout, const float* out, const float* norm, float* dk, int D, int L,
                                 void* stream);

/* ---- block glue: residual add + LayerNorm (SURVEY.md S8 f1) ---------------------------------------
 * replaces the dropout(p=0) -> add -> LayerNorm step of the pre-norm Block that wraps the mixer
 * (flash-attention/flash_attn/modules/block.py:111-148; with fused_dropout_add_ln it is
 * flash_attn.ops.layer_norm.dropout_add_layer_norm(..., prenorm=True, residual_in_fp32=True)):
 *   res_out = x + res (res may be NULL: first block, res_out may then be NULL too)
 *   y = (res_out - mean) * rstd * w + b      per row of D features, fp32; mean / rstd (rows) are saved for the backward
 * bwd: dy = grad of y, dres = grad arriving on res_out (may be NULL), r = res_out of the forward (x itself when no
 *   residual was added).  dx (rows, D) is the gradient of x AND of res; dw / db (D) are overwritten (db may be NULL).
 *   scratch: hyena_b200_add_layernorm_scratch_bytes(rows, D) bytes of per-CTA partial sums (deterministic reduction). */
HY_API size_t hyena_b200_add_layernorm_scratch_bytes(long long rows, int D);
HY_API int hyena_b200_add_layernorm_fwd(const float* x, const float* res, const float* w, const float* b, float eps,
                                 float* res_out, float* y, float* mean, float* rstd, long long rows, int D, void* stream);
HY_API int hyena_b200_add_layernorm_bwd(const float* dy, const float* dres, const float* r, const float* w, const float* mean,
                                 const float* rstd, float* dx, float* dw, float* db, long long rows, int D, void* scratch,
                                 size_t scratch_bytes, void* stream);

/* ---- incremental decoding of the causal operator -------------------------------------------------
 * The reference leaves HyenaOperator.recurrence unimplemented (hyena.py:384-386).  Output t of recurrence o is
 *     out_o[t] = sum_{s<=t} k_o[t-s] g_o[s] + fbias_o g_o[t],   g_o = v_o * x_{O-1-o},  v_0 = short(v),  v_{o+1} = out_o,
 * and y_pre[t] = out_{O-2}[t] * x_0[t] (hyena.py:404-432, filter channels ordered (d o), :408-412).  O = order, C = (O+1) D,
 * F = (O-1) D, Lcap = positions the cache holds (<= 2^20), ld = Lcap rounded up to a multiple of 4.  Cache buffers:
 *   k     F * ld + 4 floats, 16-byte aligned: filter row c time-reversed, k_c[j] at k[c*ld + ld-1-j] (padding zero)
 *   fbias (F) effective filter bias (0 * bias when use_bias is false)
 *   h     (O-1, B, D, ld), 16-byte aligned: g_o by position       tail (B, C, 2): in_proj outputs (with bias) of the last two positions
 *   s_t   (B, C) short-filter outputs of the current position      part (B, D, ceil(Lcap/1024)) scratch of one step
 * cache_B is the batch size the cache was allocated for; a different B fails.
 *   decode_hist: after a prefill of P positions, p (B, C, P) channel-major WITHOUT in_proj.bias (as for core_fwd):
 *                g_0[0..P) -> h (recurrence 0's rows) and the tail.  Later recurrences' history is copied in by the caller.
 *   decode_step: recurrence o of position t < Lcap.  o = 0 takes p_t (B, C) (in_proj output of position t without its
 *                bias), runs the short filter from the tail, writes s_t and shifts the tail; v_in must be NULL.  o > 0 takes
 *                v_in (B, D) = out of recurrence o-1.  h points at recurrence o's rows; g_o[t] is written there.  out (B, D)
 *                = out_o[t], times x_0[t] for the last recurrence (= y_pre[t]).  Two launches (one at t = 0): a split dot
 *                product over the history into part, then a fixed-order reduction and the epilogue; deterministic. */
HY_API int hyena_b200_decode_hist(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                  float* tail, int B, int cache_B, int D, int order, int P, int Lcap, void* stream);
HY_API int hyena_b200_decode_step(const float* p_t, const float* in_bias, const float* sw, const float* sb, const float* k,
                                  const float* fbias, float* h, float* tail, float* s_t, const float* v_in, float* out,
                                  float* part, int B, int cache_B, int D, int order, int o, int t, int Lcap, void* stream);
/*   decode_win_step: decode_step at a position t inside an open window [b, b + Wc) (b a multiple of 4, b + Wc <= Lcap,
 *                win (B, D, W) with W >= Wc: recurrence o's F[j] = sum_{s<b} k_o[b+j-s] g_o[s] for j < Wc, computed
 *                beforehand).  Reads the history at [b, t) only: out_o[t] = F[t-b] + sum_{b<=s<t} k_o[t-s] g_o[s]
 *                + (k_o[0] + bias_o) g_o[t].  Two launches (one at t = b); deterministic.  Same arguments otherwise. */
HY_API int hyena_b200_decode_win_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const float* win, int B, int cache_B,
                                      int D, int order, int o, int t, int b, int Wc, int W, int Lcap, void* stream);

/* ---- extending a decode cache by n >= 1 positions [t, t+n), t + n <= Lcap (chunked prefill, continuation scoring) ----
 *   decode_extend_hist:    p (B, C, n) in_proj output of the n positions WITHOUT in_proj.bias -> s (B, C, n) short-filter
 *                          outputs (carried in from the tail), g_0[t, t+n) -> h (recurrence 0's rows); shifts the tail.
 *   decode_extend_groups:  the partial count per output of decode_extend_dot for (B, D, t, n) (0 for a bad shape).
 *   decode_extend_dot:     direct Toeplitz product of recurrence o: part (B, D, n, groups), summed over groups =
 *                          sum_{s<=t+j} k_o[t+j-s] g_o[s] over h[0, t+n), which must already hold g_o of the n positions.
 *   decode_extend_combine: out_o[t+j] = sum_g part[row * row_stride + j * j_stride + g] + fbias_o g_o[t+j], times the gate
 *                          s[(O-2-o) D + d][j]: into the rows of recurrence o+1 (out = its h) or, for the last recurrence,
 *                          y_pre (B, D, n) (out).  part may also be a full convolution (groups 1: the FFT route).
 * Deterministic: fixed summation orders, no atomics. */
HY_API int hyena_b200_decode_extend_groups(int B, int D, int t, int n);
HY_API int hyena_b200_decode_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb, float* h,
                                         float* tail, float* s, int B, int cache_B, int D, int order, int t, int n, int Lcap,
                                         void* stream);
HY_API int hyena_b200_decode_extend_dot(const float* h, const float* k, float* part, int groups, int B, int cache_B, int D,
                                        int order, int o, int t, int n, int Lcap, void* stream);
HY_API int hyena_b200_decode_extend_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out, int B,
                                            int cache_B, int D, int order, int o, int t, int n, int Lcap, void* stream);

/* ---- decoding a branched cache (R branches forked from one context at base b, a multiple of 4) ----
 * Each of the R rows of h (recurrence o's rows, 16-byte aligned) holds g_o of positions [b, b + Hc) of one branch with row
 * stride H (a multiple of 4, Hc <= H <= ld - b, b + Hc <= Lcap); tail, s_t, s, part and out have R rows.  k and fbias are the
 * parent cache's (ld = Lcap rounded up to a multiple of 4).  f (P, D, H) holds recurrence o's F[p][d][j] =
 * sum_{s<b} k_o[b+j-s] g_o[s] of parent row p for j < Hc; parent (R) int32 on the device gives the F row of each branch
 * (not checked here: every entry must be in [0, P)).  Positions t are absolute; t and t + n must stay in [b, b + Hc).
 *   decode_branch_step:        decode_step of position t on the branches: out_o[t] = F[parent][t-b]
 *                              + sum_{b<=s<t} k_o[t-s] g_o[s] + (k_o[0] + bias_o) g_o[t].  Two launches (one at t = b).
 *   decode_branch_extend_hist: decode_extend_hist of the n positions [t, t+n) on the branch rows.
 *   decode_branch_extend_dot:  decode_extend_dot over the branch positions [b, t+n): part (R, D, n, groups) with groups =
 *                              decode_extend_groups(R, D, t - b, n).
 *   decode_branch_combine:     decode_extend_combine + F[parent][t-b+j]; part may also be the FFT route's convolution of the
 *                              branch rows (positions from b on).
 * Deterministic: fixed summation orders, no atomics. */
HY_API int hyena_b200_decode_branch_step(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                         const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                         const float* v_in, float* out, float* part, const float* f, const int* parent,
                                         int R, int D, int order, int o, int t, int b, int Hc, int H, int Lcap,
                                         void* stream);
HY_API int hyena_b200_decode_branch_extend_hist(const float* p, const float* in_bias, const float* sw, const float* sb,
                                                float* h, float* tail, float* s, int R, int D, int order, int t, int n,
                                                int b, int Hc, int H, int Lcap, void* stream);
HY_API int hyena_b200_decode_branch_extend_dot(const float* h, const float* k, float* part, int groups, int R, int D,
                                               int order, int o, int t, int n, int b, int Hc, int H, int Lcap,
                                               void* stream);
HY_API int hyena_b200_decode_branch_combine(const float* part, long long row_stride, int j_stride, int groups,
                                            const float* fbias, const float* h, const float* s, float* out,
                                            const float* f, const int* parent, int R, int D, int order, int o, int t,
                                            int n, int b, int Hc, int H, int Lcap, void* stream);

/* ---- device-position steps: one step captured in a CUDA graph and replayed at every position ----
 * pos (3 int32 on the device) = [t, win_b, base]: the position, the base of the open window and the base of a branched
 * cache.  These calls read no position on the host: their kernels read pos when they run, on grids fixed by the arguments
 * (the dot kernel's CTAs past the position leave at once).  The caller keeps pos within the bounds below; a replay
 * cannot check them.  The outputs are bit-identical to the host-position calls at the same state.  They allocate nothing
 * and never synchronise, so they can be captured once the library has been used on the capturing stream.
 *   decode_step_dev:        decode_step at t = pos[0], which must stay below t_max <= Lcap (grid: ceil(t_max / 1024)
 *                           chunks).
 *   decode_win_step_dev:    decode_win_step at t = pos[0] in the window based at pos[1]: 0 <= t - pos[1] < the window's
 *                           width, which is at most W (win (B, D, W); grid: ceil(W / 1024) chunks).
 *   decode_branch_step_dev: decode_branch_step at t = pos[0] of branches based at pos[2]: t - pos[2] < Hc <= H.
 *   decode_pos_advance:     pos[0] += 1, one thread.  Enqueue it after every call of the step that reads pos.
 * Launches count under the kinds of the host-position calls; decode_pos_advance's under none (launch_count only).  While
 * a stream is being captured, the per-launch event timing (profile_begin / profile_end) skips it. */
HY_API int hyena_b200_decode_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                      const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                      const float* v_in, float* out, float* part, const int* pos, int B, int cache_B, int D,
                                      int order, int o, int t_max, int Lcap, void* stream);
HY_API int hyena_b200_decode_win_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                          const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                          const float* v_in, float* out, float* part, const float* win, const int* pos, int B,
                                          int cache_B, int D, int order, int o, int W, int Lcap, void* stream);
HY_API int hyena_b200_decode_branch_step_dev(const float* p_t, const float* in_bias, const float* sw, const float* sb,
                                             const float* k, const float* fbias, float* h, float* tail, float* s_t,
                                             const float* v_in, float* out, float* part, const float* f, const int* parent,
                                             const int* pos, int R, int D, int order, int o, int H, int Lcap, void* stream);
HY_API int hyena_b200_decode_pos_advance(int* pos, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HYENA_B200_H */
