"""Raw device ops (thin wrappers over the C ABI) and the autograd Functions built on them.

PyTorch provides device memory, streams and autograd plumbing; all arithmetic of the custom-kernel
span runs in libhyena_b200.so.  Inputs must be CUDA fp32 tensors -- anything else raises.
"""
import contextlib

import torch

from . import _lib

_ws_cache = {}


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.HyenaB200Error("hyena_b200 ops need CUDA tensors (there is no CPU path)")
        if t.dtype != torch.float32:
            raise _lib.HyenaB200Error(f"hyena_b200 ops compute in fp32; got {t.dtype}")


def workspace(B, D, L, backward, device):
    """Cached scratch buffer for the FFT passes, one per (device, stream): two operators driven from different streams
    (DDP bucket hooks, checkpoint recompute on a side stream) never share scratch, so the op stays re-entrant across
    streams as the reference extension is (csrc/fftconv/fftconv.cpp allocates per call)."""
    n = int(_lib.lib().hyena_b200_workspace_bytes(B, D, L, int(backward)))
    key = (device.index if device.index is not None else torch.cuda.current_device(), _stream())
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < n:
        buf = torch.empty(n, dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    # hand the library exactly the bytes this call asked for: the group size (rows in flight, sized to
    # stay L2-resident) is derived from the workspace size
    return buf[:n]


def spectrum_elems(L):
    return int(_lib.lib().hyena_b200_spectrum_elems(int(L)))


# ------------------------------------------------------------------------------------------ filter
def _filter_args(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L):
    E = z.shape[-1]
    N = W1.shape[0]
    D = W3.shape[0]
    rows = z.shape[-2]
    if L < 1 or L > rows or L > t.shape[-2 if t.dim() == 3 else 0]:
        raise _lib.HyenaB200Error(f"filter length {L} exceeds the positional embedding ({rows} rows); the reference "
                                  "returns a seq_len-long filter, callers clamp with min(L, l_max)")
    zz = z[0, :L] if z.dim() == 3 else z[:L]
    tt = (t[0, :L, 0] if t.dim() == 3 else t[:L]).contiguous()
    if zz.stride(-1) != 1:
        zz = zz.contiguous()
    return zz, tt, E, N, D


def filter_forward(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L):
    """k (D, L) channel-major == HyenaFilter.filter(L)[0].T  (hyena.py:229-238)."""
    _need_cuda(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas)
    zz, tt, E, N, D = _filter_args(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L)
    k = torch.empty(D, L, dtype=torch.float32, device=z.device)
    ws = [x.contiguous() for x in (W0, b0, W1, b1, W2, b2, W3)]
    fr = freq.reshape(-1).contiguous()
    dl = deltas.reshape(-1).contiguous()
    with torch.cuda.device(z.device):
        _lib.check(_lib.lib().hyena_b200_filter_fwd(
            _ptr(zz), zz.stride(0), _ptr(tt), *[_ptr(w) for w in ws], _ptr(fr), _ptr(dl),
            float(shift), int(bool(modulate)), int(L), E, N, D, _ptr(k), _stream()))
    return k


def _filter_backward_tc(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, dk, need_dz):
    """Tensor-core backward: stage 1 on wgmma (csrc/filter_tc.cuh), stage 2 = sequence-length reductions."""
    zz, tt, E, N, D = _filter_args(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L)
    ws = [x.contiguous() for x in (W0, b0, W1, b1, W2, b2, W3)]
    fr = freq.reshape(-1).contiguous()
    dl = deltas.reshape(-1).contiguous()
    dk = dk.contiguous()
    dev = z.device
    dh = torch.empty(D, L, dtype=torch.float32, device=dev)
    sc = torch.empty(7, 64, L, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hyena_b200_filter_bwd_stage1(
            _ptr(zz), zz.stride(0), _ptr(tt), *[_ptr(w) for w in ws], _ptr(fr), _ptr(dl),
            float(shift), int(bool(modulate)), int(L), E, N, D, _ptr(dk), _ptr(dh), _ptr(sc), _stream()))
    a1, a2, a3, dp1, dp2, dp3, X = sc.unbind(0)          # feature-major (64, L) each
    if D <= 256 and E <= 8:
        grads = [torch.zeros_like(w) for w in ws]
        dfreq = torch.zeros(64, dtype=torch.float32, device=dev)
        zT = zz.t().contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hyena_b200_filter_bwd_stage2(
                _ptr(dh), _ptr(sc), _ptr(zT), *[_ptr(g) for g in grads], _ptr(dfreq), int(L), E, D, _stream()))
    else:                                             # wide models: library GEMMs with K = L
        sums = sc[3:7].sum(dim=2)
        grads = [dp1 @ zz, sums[0], dp2 @ a1.t(), sums[1], dp3 @ a2.t(), sums[2], dh @ a3.t()]
        dfreq = sums[3]
    dz = (dp1.t() @ ws[0]) if need_dz else None
    return grads, dfreq, dz


def filter_backward(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, dk, need_dz):
    _need_cuda(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, dk)
    import os
    if os.environ.get("HYENA_B200_FILTER", "tc") != "simt":
        return _filter_backward_tc(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, dk, need_dz)
    zz, tt, E, N, D = _filter_args(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L)
    ws = [x.contiguous() for x in (W0, b0, W1, b1, W2, b2, W3)]
    fr = freq.reshape(-1).contiguous()
    dl = deltas.reshape(-1).contiguous()
    dk = dk.contiguous()
    grads = [torch.zeros_like(w) for w in ws]
    dfreq = torch.zeros_like(fr)
    dz = torch.zeros(L, E, dtype=torch.float32, device=z.device) if need_dz else None
    with torch.cuda.device(z.device):
        _lib.check(_lib.lib().hyena_b200_filter_bwd(
            _ptr(zz), zz.stride(0), _ptr(tt), *[_ptr(w) for w in ws], _ptr(fr), _ptr(dl),
            float(shift), int(bool(modulate)), int(L), E, N, D, _ptr(dk),
            *[_ptr(g) for g in grads], _ptr(dfreq), _ptr(dz), E, _stream()))
    return grads, dfreq, dz


class HyenaFilterFn(torch.autograd.Function):
    """Differentiable implicit filter: parameters -> k (D, L)."""

    @staticmethod
    def forward(ctx, z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L, cached=None):
        ctx.cfg = (shift, modulate, L)
        if cached is not None:                 # same inputs as the call that produced it (HyenaFilter.filter_channel_major)
            k = cached.detach()
        else:
            k = filter_forward(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L)
        # trainable deltas (modulation_lr != 0): their gradient needs the filter itself
        need_k = modulate and torch.is_tensor(deltas) and deltas.requires_grad
        ctx.save_for_backward(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, k if need_k else None)
        return k

    @staticmethod
    def backward(ctx, dk):
        z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, ksaved = ctx.saved_tensors
        shift, modulate, L = ctx.cfg
        ddelta = None
        if ctx.needs_input_grad[10]:
            if not modulate or ksaved is None:
                ddelta = torch.zeros_like(deltas)
            else:                                      # ExponentialModulation with modulation_lr != 0 (hyena.py:145-155)
                D = ksaved.shape[0]
                dkc = dk.contiguous()
                tt = (t[0, :L, 0] if t.dim() == 3 else t[:L]).contiguous()
                dl = deltas.reshape(-1).contiguous()
                dd = torch.empty(D, dtype=torch.float32, device=dk.device)
                with torch.cuda.device(dk.device):
                    _lib.check(_lib.lib().hyena_b200_filter_ddelta(_ptr(dkc), _ptr(ksaved), _ptr(tt), _ptr(dl), float(shift),
                                                                    D, int(L), _ptr(dd), _stream()))
                ddelta = dd.reshape(deltas.shape)
        need_dz = ctx.needs_input_grad[0]
        grads, dfreq, dz = filter_backward(z, t, W0, b0, W1, b1, W2, b2, W3, freq, deltas, shift, modulate, L,
                                           dk, need_dz)
        gz = None
        if need_dz:
            gz = torch.zeros_like(z)
            (gz[0, :L] if z.dim() == 3 else gz[:L]).copy_(dz)
        return (gz, None, *grads, dfreq.reshape(freq.shape), ddelta, None, None, None, None)


class FilterL1NormFn(torch.autograd.Function):
    """k (D, L) -> k / sum_c |k[c, t]|: HyenaFilter(normalized=True), hyena.py:235-236 (L1 norm over the channel dim of the
    reference's (1, L, D) layout)."""

    @staticmethod
    def forward(ctx, k):
        _need_cuda(k)
        k = k.contiguous()
        D, L = k.shape
        out = torch.empty_like(k)
        norm = torch.empty(L, dtype=torch.float32, device=k.device)
        with torch.cuda.device(k.device):
            _lib.check(_lib.lib().hyena_b200_filter_l1norm_fwd(_ptr(k), _ptr(out), _ptr(norm), D, L, _stream()))
        ctx.save_for_backward(out, norm)
        return out

    @staticmethod
    def backward(ctx, dout):
        out, norm = ctx.saved_tensors
        dout = dout.contiguous()
        _need_cuda(dout)
        D, L = out.shape
        dk = torch.empty_like(out)
        with torch.cuda.device(out.device):
            _lib.check(_lib.lib().hyena_b200_filter_l1norm_bwd(_ptr(dout), _ptr(out), _ptr(norm), _ptr(dk), D, L, _stream()))
        return dk


# ------------------------------------------------------------------------------------------ spectrum / core
def filter_spectrum(k):
    """Opaque packed spectrum of k (D, L) -> (D, M) complex64 (replaces rfft(k, 2L)/2L, hyena.py:62)."""
    _need_cuda(k)
    k = k.contiguous()
    D, L = k.shape
    M = spectrum_elems(L)
    spec = torch.empty(D, M, dtype=torch.complex64, device=k.device)
    ws = workspace(1, D, L, False, k.device)
    with torch.cuda.device(k.device):
        _lib.check(_lib.lib().hyena_b200_filter_spectrum(_ptr(k), _ptr(spec), D, L, _ptr(ws), ws.numel(), _stream()))
    return spec


def _check_spectrum(kspec, H, L, what):
    """The packed spectrum is opaque but its type and shape are not: (H, spectrum_elems(L)) complex64, contiguous, on the
    same device -- anything else (e.g. the reference's rfft(k, fft_size), src/ops/fftconv.py:65) would be read out of
    bounds or silently misinterpreted by the kernels."""
    M = spectrum_elems(L)
    if not (torch.is_tensor(kspec) and kspec.is_cuda and kspec.dtype == torch.complex64 and kspec.dim() == 2
            and tuple(kspec.shape) == (H, M) and kspec.is_contiguous()):
        got = (tuple(kspec.shape), kspec.dtype) if torch.is_tensor(kspec) else type(kspec)
        raise _lib.HyenaB200Error(f"{what}: filter spectrum must be the packed form from filter_spectrum(): contiguous "
                                  f"complex64 ({H}, {M}) on the GPU; got {got}.  For the reference's rfft(k, fft_size) "
                                  "use fftconv.fftconv_fwd / fftconv_bwd, which convert it")


def spectrum_from_rfft(filt, L, fft_size):
    """rfft(k, n=fft_size) (H, fft_size/2+1) complex64 -- the filter the reference extension takes
    (src/ops/fftconv.py:64-65) -- to the packed spectrum the kernels consume."""
    if not (torch.is_tensor(filt) and filt.is_cuda and filt.dtype == torch.complex64 and filt.dim() == 2
            and filt.shape[1] == fft_size // 2 + 1):
        raise _lib.HyenaB200Error(f"filter must be a CUDA complex64 (H, fft_size/2+1 = {fft_size // 2 + 1}) tensor")
    filt = filt.contiguous()
    H = filt.shape[0]
    M = spectrum_elems(L)
    spec = torch.empty(H, M, dtype=torch.complex64, device=filt.device)
    ksc = torch.empty(H, L, dtype=torch.float32, device=filt.device) if fft_size < 2 * M else None
    ws = workspace(1, H, L, False, filt.device)
    with torch.cuda.device(filt.device):
        _lib.check(_lib.lib().hyena_b200_spectrum_from_rfft(_ptr(filt), int(fft_size), _ptr(spec), _ptr(ksc), H, int(L),
                                                            _ptr(ws), ws.numel(), _stream()))
    return spec


def spectrum_to_rfft(dk, fft_size):
    """dk (H, L) time domain -> dfilter (H, fft_size/2+1) complex64 with irfft(dfilter, n=fft_size, norm='forward')[:L]
    == dk: what csrc/fftconv/fftconv.cpp:235 returns and src/ops/fftconv.py:98 consumes."""
    _need_cuda(dk)
    dk = dk.contiguous()
    H, L = dk.shape
    M = spectrum_elems(L)
    out = torch.empty(H, fft_size // 2 + 1, dtype=torch.complex64, device=dk.device)
    ssc = torch.empty(H, M, dtype=torch.complex64, device=dk.device) if fft_size == 2 * M else None
    ws = workspace(1, H, L, False, dk.device)
    with torch.cuda.device(dk.device):
        _lib.check(_lib.lib().hyena_b200_spectrum_to_rfft(_ptr(dk), int(fft_size), _ptr(out), _ptr(ssc), H, int(L),
                                                          _ptr(ws), ws.numel(), _stream()))
    return out


def _save_spectrum():
    import os
    return os.environ.get("HYENA_B200_SAVE_SPECTRUM", "1") != "0"


def core_forward(p, in_bias, sw, sb, kspec, fbias, save_c):
    _need_cuda(p, in_bias, sw, sb, fbias)
    B, C3, L = p.shape
    D = C3 // 3
    if C3 != 3 * D or not p.is_contiguous():
        raise _lib.HyenaB200Error("core_forward: p must be contiguous (B, 3D, L)")
    _check_spectrum(kspec, D, L, "core_forward")
    if sw.numel() != 3 * C3 or sb.numel() != C3 or fbias.numel() != D or (in_bias is not None and in_bias.numel() != C3):
        raise _lib.HyenaB200Error("core_forward: short filter / bias shapes do not match p")
    y = torch.empty(B, D, L, dtype=torch.float32, device=p.device)
    c = torch.empty(B, D, L, dtype=torch.float32, device=p.device) if save_c else None
    # spectrum of the gated input, rows ordered (c, b): saves a column pass + a row FFT per row in backward
    gs = (torch.empty(D * B, kspec.shape[-1], dtype=torch.complex64, device=p.device)
          if (save_c and _save_spectrum()) else None)
    ws = workspace(B, D, L, False, p.device)
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().hyena_b200_core_fwd(
            _ptr(p), _ptr(in_bias), _ptr(sw), _ptr(sb), _ptr(kspec), _ptr(fbias), _ptr(y), _ptr(c), _ptr(gs),
            B, D, L, _ptr(ws), ws.numel(), _stream()))
    return y, c, gs


def core_backward(dy_pre, p, in_bias, sw, sb, kspec, fbias, c_saved, gspec=None, return_ds=False):
    _need_cuda(dy_pre, p, in_bias, sw, sb, fbias, c_saved)
    B, C3, L = p.shape
    D = C3 // 3
    dev = p.device
    _check_spectrum(kspec, D, L, "core_backward")
    if tuple(dy_pre.shape) != (B, D, L) or tuple(c_saved.shape) != (B, D, L):
        raise _lib.HyenaB200Error("core_backward: dy_pre / c_saved must be (B, D, L)")
    dy_pre = dy_pre.contiguous()
    dp = None if return_ds else torch.empty_like(p)
    ds = torch.empty_like(p)
    dk = torch.empty(D, L, dtype=torch.float32, device=dev)
    dsw = torch.zeros(C3, 3, dtype=torch.float32, device=dev)
    dsb = torch.zeros(C3, dtype=torch.float32, device=dev)
    dfb = torch.zeros(D, dtype=torch.float32, device=dev)
    dib = torch.zeros(C3, dtype=torch.float32, device=dev) if in_bias is not None else None
    ws = workspace(B, D, L, True, dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hyena_b200_core_bwd(
            _ptr(dy_pre), _ptr(p), _ptr(in_bias), _ptr(sw), _ptr(sb), _ptr(kspec), _ptr(fbias), _ptr(c_saved),
            _ptr(gspec), _ptr(dp), _ptr(dk), _ptr(dsw), _ptr(dsb), _ptr(dfb), _ptr(dib), _ptr(ds),
            B, D, L, _ptr(ws), ws.numel(), _stream()))
    if return_ds:
        # d in_proj.bias = sum_t dp[t] = (w0 + w1 + w2) sum_t ds[t] - w1 ds[0] - w0 (ds[0] + ds[1])   (conv padding edge)
        if in_bias is not None:
            e0 = ds[:, :, 0].sum(0)
            e1 = ds[:, :, 1].sum(0) if L > 1 else torch.zeros_like(e0)
            dib = sw.sum(1) * dsb - sw[:, 1] * e0 - sw[:, 0] * (e0 + e1)
        return ds, dk, dsw, dsb, dfb, dib
    del ds
    return dp, dk, dsw, dsb, dfb, dib


class HyenaCoreFn(torch.autograd.Function):
    """(p, in_bias, short filter, k, filter bias) -> y_pre (B, D, L); hyena.py:394-432 for order 2."""

    @staticmethod
    def forward(ctx, p, in_bias, sw, sb, k, fbias, kspec=None):
        p = p.contiguous()
        sw2 = sw.reshape(sw.shape[0], -1).contiguous()
        sb = sb.contiguous(); fbias = fbias.contiguous()
        ib = in_bias.contiguous() if in_bias is not None else None
        if kspec is None:
            kspec = filter_spectrum(k)
        need = any(ctx.needs_input_grad)
        y, c, gs = core_forward(p, ib, sw2, sb, kspec, fbias, need)
        ctx.save_for_backward(p, ib, sw2, sb, kspec, fbias, c, gs)
        ctx.sw_shape = sw.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        p, ib, sw2, sb, kspec, fbias, c, gs = ctx.saved_tensors
        dp, dk, dsw, dsb, dfb, dib = core_backward(dy, p, ib, sw2, sb, kspec, fbias, c, gs)
        return dp, dib, dsw.reshape(ctx.sw_shape), dsb, dk, dfb, None


class HyenaInCoreFn(torch.autograd.Function):
    """in_proj + operator core as ONE autograd node (wgmma projections): u (B, L, D) -> y_pre (B, D, L).

    Forward: p = W u^T channel-major (proj_gemm), then the fused core.  Backward: the core returns ds (gradient w.r.t. the
    short-filter outputs) and the two projection-backward GEMMs apply the transposed 3-tap filter to it on the fly, so
    neither dp nor a separate short-filter backward pass exists (hyena.py:391-432 and its autograd)."""

    @staticmethod
    def forward(ctx, u, W, in_bias, sw, sb, k, fbias, kspec=None):
        u = u.contiguous(); W = W.contiguous()
        sw2 = sw.reshape(sw.shape[0], -1).contiguous()
        sb = sb.contiguous(); fbias = fbias.contiguous()
        ib = in_bias.contiguous() if in_bias is not None else None
        p = proj_gemm(u, 0, W, False, 0)
        if kspec is None:
            kspec = filter_spectrum(k)
        need = any(ctx.needs_input_grad)
        y, c, gs = core_forward(p, ib, sw2, sb, kspec, fbias, need)
        ctx.save_for_backward(u, W, p, ib, sw2, sb, kspec, fbias, c, gs)
        ctx.sw_shape = sw.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        u, W, p, ib, sw2, sb, kspec, fbias, c, gs = ctx.saved_tensors
        ds, dk, dsw, dsb, dfb, dib = core_backward(dy, p, ib, sw2, sb, kspec, fbias, c, gs, return_ds=True)
        du = proj_gemm(ds, 1, W, True, 1, fir=sw2) if ctx.needs_input_grad[0] else None
        dW = proj_wgrad(ds, u, fir=sw2) if ctx.needs_input_grad[1] else None
        return du, dW, dib, dsw.reshape(ctx.sw_shape), dsb, dk, dfb, None


# ------------------------------------------------------------------------------------------ plain fftconv
def fftconv_forward(u, kspec, Dvec):
    _need_cuda(u, Dvec)
    if u.dim() != 3 or not u.is_contiguous():
        raise _lib.HyenaB200Error("fftconv_forward: u must be contiguous (B, H, L)")
    B, H, L = u.shape
    _check_spectrum(kspec, H, L, "fftconv_forward")
    if Dvec.numel() != H or not Dvec.is_contiguous():
        raise _lib.HyenaB200Error(f"fftconv_forward: D must have {H} contiguous elements, got {tuple(Dvec.shape)}")
    out = torch.empty_like(u)
    ws = workspace(B, H, L, False, u.device)
    with torch.cuda.device(u.device):
        _lib.check(_lib.lib().hyena_b200_fftconv_fwd(_ptr(u), _ptr(kspec), _ptr(Dvec), _ptr(out), B, H, L,
                                                     _ptr(ws), ws.numel(), _stream()))
    return out


def fftconv_backward(dout, u, kspec, Dvec):
    _need_cuda(dout, u, Dvec)
    if u.dim() != 3 or not u.is_contiguous() or tuple(dout.shape) != tuple(u.shape) or not dout.is_contiguous():
        raise _lib.HyenaB200Error("fftconv_backward: u and dout must be contiguous (B, H, L) of the same shape")
    B, H, L = u.shape
    _check_spectrum(kspec, H, L, "fftconv_backward")
    if Dvec.numel() != H or not Dvec.is_contiguous():
        raise _lib.HyenaB200Error(f"fftconv_backward: D must have {H} contiguous elements, got {tuple(Dvec.shape)}")
    du = torch.empty_like(u)
    dk = torch.empty(H, L, dtype=torch.float32, device=u.device)
    dD = torch.zeros(H, dtype=torch.float32, device=u.device)
    ws = workspace(B, H, L, True, u.device)
    with torch.cuda.device(u.device):
        _lib.check(_lib.lib().hyena_b200_fftconv_bwd(_ptr(dout), _ptr(u), _ptr(kspec), _ptr(Dvec), _ptr(du), _ptr(dk),
                                                     _ptr(dD), B, H, L, _ptr(ws), ws.numel(), _stream()))
    return du, dk, dD


# ------------------------------------------------------------------------------------------ projections
_gemm_ws = {}
_gemm_mode = None


def gemm_mode():
    """'bf16x9' when the CUDA 12.9 cuBLASLt with fp32 emulation is usable, else 'torch' (torch.bmm on the
    bundled cuBLAS).  HYENA_B200_GEMM=torch forces the latter.  Both are GPU library GEMMs."""
    global _gemm_mode
    if _gemm_mode is None:
        import os
        want = os.environ.get("HYENA_B200_GEMM", "bf16x9")
        _gemm_mode = "torch"
        if want != "torch" and torch.cuda.is_available() and _lib.lib().hyena_b200_gemm_available():
            _gemm_mode = "bf16x9"
    return _gemm_mode


def gemm(transa, transb, m, n, k, A, lda, strideA, B, ldb, strideB, C, ldc, strideC, batch=1, beta=0.0, bias=None,
         emulate=None):
    """Column-major strided-batched C = op(A) op(B) + beta*C (+bias) on cuBLASLt 12.9 (see csrc/gemm.cu).

    Precision follows PyTorch's own switch, like the reference's nn.Linear does: fp32-accurate BF16x9 emulation by
    default, TF32 tensor cores when the user set ``torch.backends.cuda.matmul.allow_tf32 = True`` (the reference
    training script does, train.py:34-35)."""
    if emulate is None:
        emulate = 2 if torch.backends.cuda.matmul.allow_tf32 else 1
    dev = C.device
    # one workspace per (device, stream): GEMMs issued on different streams may run concurrently
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), _stream())
    ws = _gemm_ws.get(key)
    if ws is None:
        ws = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
        _gemm_ws[key] = ws
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hyena_b200_gemm(int(transa), int(transb), m, n, k, 1.0, _ptr(A), lda, strideA,
                                              _ptr(B), ldb, strideB, float(beta), _ptr(C), ldc, strideC, batch,
                                              _ptr(bias), int(emulate), _ptr(ws), ws.numel(), _stream()))
    return C


_wimg_cache = {}
_proj_mode = None


def proj_mode():
    """'tc': the projections run on this library's wgmma 3xTF32 kernels (csrc/proj_gemm.cuh) -- the default;
    'lt': cuBLASLt 12.9 BF16x9 (csrc/gemm.cu; also what runs when the user opted into TF32 via
    torch.backends.cuda.matmul.allow_tf32); 'torch': torch.bmm.  HYENA_B200_PROJ selects."""
    global _proj_mode
    if _proj_mode is None:
        import os
        want = os.environ.get("HYENA_B200_PROJ", "tc")
        if want == "tc":
            _proj_mode = "tc"
        else:
            _proj_mode = "lt" if (want != "torch" and gemm_mode() == "bf16x9") else "torch"
    if _proj_mode == "tc" and torch.backends.cuda.matmul.allow_tf32 and gemm_mode() == "bf16x9":
        return "lt"          # plain-TF32 opt-in: one MMA per product on the library path
    return _proj_mode


_GELU_CODES = {"tanh": 1, "none": 2}        # F.gelu(approximate=...) -> HYENA_B200_GELU_TANH / HYENA_B200_GELU_ERF


def _gelu_code(approximate):
    if approximate not in _GELU_CODES:
        raise _lib.HyenaB200Error(f"GELU approximate must be 'tanh' or 'none', got {approximate!r}")
    return _GELU_CODES[approximate]


@contextlib.contextmanager
def private_weight_images(device, stream, keep):
    """proj_gemm calls on ``stream`` inside the block use weight-image scratch of their own instead of the shared
    per-stream entry of _wimg_cache, and that scratch is appended to ``keep``.  For CUDA-graph capture: a graph bakes the
    scratch address in, while the shared entry can be replaced (and its memory freed) by any later, larger call on a stream
    with the same handle (torch hands out pooled streams).  The shared entry is restored afterwards."""
    key = (device.index if device.index is not None else torch.cuda.current_device(), stream.cuda_stream)
    shared = _wimg_cache.pop(key, None)
    try:
        yield
    finally:
        own = _wimg_cache.pop(key, None)
        if own is not None:
            keep.append(own)
        if shared is not None:
            _wimg_cache[key] = shared


def proj_gemm(act, act_layout, W, w_transposed, out_layout, bias=None, fir=None, out=None, l_range=None, gelu=None,
              gelu_pre=None):
    """OUT[pos][n] = sum_k ACT[pos][k] Wl[n][k] (+ bias) on this library's wgmma kernel (csrc/proj_gemm.cuh, 3xTF32).
    act_layout 0: act (B, L, K); 1: act (B, K, L).  out_layout 0: (B, N, L); 1: (B, L, N).  Wl = W.T if w_transposed.

    gelu ('tanh' | 'none', F.gelu's ``approximate``) fuses the block MLP's activation: with act_layout 1 / out_layout 1 the
    GEMM consumes gelu(act); with act_layout 0 / out_layout 0 and ``gelu_pre`` (B, N, L) the output is multiplied by
    gelu'(gelu_pre)."""
    _need_cuda(act, W, bias, fir, gelu_pre)
    if act.dim() != 3 or W.dim() != 2 or not act.is_contiguous() or not W.is_contiguous():
        raise _lib.HyenaB200Error("proj_gemm: act must be contiguous 3-D, W contiguous 2-D")
    B = act.shape[0]
    L, K = (act.shape[1], act.shape[2]) if act_layout == 0 else (act.shape[2], act.shape[1])
    N = W.shape[1] if w_transposed else W.shape[0]
    if (W.shape[0] if w_transposed else W.shape[1]) != K:
        raise _lib.HyenaB200Error(f"proj_gemm: weight {tuple(W.shape)} does not match K = {K}")
    dev = act.device
    oshape = (B, N, L) if out_layout == 0 else (B, L, N)
    if out is None:
        out = torch.empty(oshape, dtype=torch.float32, device=dev)
    elif tuple(out.shape) != oshape or not out.is_contiguous() or out.dtype != torch.float32:
        raise _lib.HyenaB200Error(f"proj_gemm: out must be contiguous fp32 {oshape}")
    l0, ln = (0, 0) if l_range is None else (int(l_range[0]), int(l_range[1] - l_range[0]))
    need = int(_lib.lib().hyena_b200_proj_wimg_bytes(N, K))
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), _stream())
    wimg = _wimg_cache.get(key)
    if wimg is None or wimg.numel() < need:
        wimg = torch.empty(max(need, 4 << 20), dtype=torch.uint8, device=dev)
        _wimg_cache[key] = wimg
    if gelu is not None:
        code = _gelu_code(gelu)
        if fir is not None or l_range is not None:
            raise _lib.HyenaB200Error("proj_gemm: the fused GELU takes no short filter and no position range")
        if act_layout == 1 and out_layout == 1 and gelu_pre is None:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().hyena_b200_proj_gemm_gelu(
                    _ptr(act), _ptr(W), W.shape[1], int(bool(w_transposed)), _ptr(bias), code, _ptr(out), B, L, K, N,
                    _ptr(wimg), wimg.numel(), _stream()))
            return out
        if act_layout == 0 and out_layout == 0 and bias is None and gelu_pre is not None:
            if tuple(gelu_pre.shape) != oshape or not gelu_pre.is_contiguous():
                raise _lib.HyenaB200Error(f"proj_gemm: gelu_pre must be contiguous {oshape}")
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().hyena_b200_proj_gemm_dgelu(
                    _ptr(act), _ptr(W), W.shape[1], int(bool(w_transposed)), _ptr(gelu_pre), code, _ptr(out), B, L, K, N,
                    _ptr(wimg), wimg.numel(), _stream()))
            return out
        raise _lib.HyenaB200Error("proj_gemm: the fused GELU runs as (act_layout 1, out_layout 1) or, with gelu_pre and "
                                  "no bias, as (act_layout 0, out_layout 0)")
    if gelu_pre is not None:
        raise _lib.HyenaB200Error("proj_gemm: gelu_pre needs gelu")
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().hyena_b200_proj_gemm(
            _ptr(act), int(act_layout), _ptr(W), W.shape[1], int(bool(w_transposed)), _ptr(bias), _ptr(fir), _ptr(out),
            int(out_layout), B, L, K, N, l0, ln, _ptr(wimg), wimg.numel(), _stream()))
    return out


_wgrad_cache = {}


def fuse_fir():
    """Transposed short filter fused into the projection-backward GEMMs (default on; HYENA_B200_FUSE_FIR=0 keeps the
    separate short_conv_bwd pass for A/B runs)."""
    import os
    return os.environ.get("HYENA_B200_FUSE_FIR", "1") != "0"


def proj_wgrad(X, Y, fir=None, transposed_out=False, gelu=None):
    """dW (M, N) [(N, M) if transposed_out] = sum_{b,pos} X[b][m][pos] Y[b][pos][n]; X (B, M, L), Y (B, L, N)
    (csrc/proj_gemm.cuh wgrad_kernel: wgmma 3xTF32, split-K, deterministic).  gelu ('tanh' | 'none'): the product is
    taken with gelu(X) instead of X (block MLP fc2 weight gradient)."""
    _need_cuda(X, Y, fir)
    if X.dim() != 3 or Y.dim() != 3 or not X.is_contiguous() or not Y.is_contiguous() or X.shape[0] != Y.shape[0] \
            or X.shape[2] != Y.shape[1]:
        raise _lib.HyenaB200Error(f"proj_wgrad: X (B, M, L) / Y (B, L, N) expected, got {tuple(X.shape)} / {tuple(Y.shape)}")
    B, M, L = X.shape
    N = Y.shape[2]
    dev = X.device
    dW = torch.empty((N, M) if transposed_out else (M, N), dtype=torch.float32, device=dev)
    need = int(_lib.lib().hyena_b200_proj_wgrad_scratch_bytes(M, N))
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), _stream())
    sc = _wgrad_cache.get(key)
    if sc is None or sc.numel() < need:
        sc = torch.empty(need, dtype=torch.uint8, device=dev)
        _wgrad_cache[key] = sc
    with torch.cuda.device(dev):
        if gelu is not None:
            if fir is not None:
                raise _lib.HyenaB200Error("proj_wgrad: the fused GELU takes no short filter")
            _lib.check(_lib.lib().hyena_b200_proj_wgrad_gelu(_ptr(X), _ptr(Y), _gelu_code(gelu), _ptr(dW),
                                                             int(bool(transposed_out)), 0.0, B, L, M, N, _ptr(sc), sc.numel(),
                                                             _stream()))
        else:
            _lib.check(_lib.lib().hyena_b200_proj_wgrad(_ptr(X), _ptr(Y), _ptr(fir), _ptr(dW), int(bool(transposed_out)),
                                                        0.0, B, L, M, N, _ptr(sc), sc.numel(), _stream()))
    return dW


class MlpFn(torch.autograd.Function):
    """Block MLP y = fc2(gelu(fc1(x))) as ONE autograd node on the wgmma projection kernels, fp32 (3xTF32).

    Replaces flash_attn/modules/mlp.py:26-30 (the Mlp that src/models/sequence/long_conv_lm.py:102-123 builds).  x is
    (B, L, D); the hidden activation a = fc1(x) is written channel-major (B, H, L), the layout in which every GEMM of the
    MLP is one the projection kernels already run.  GELU is applied in fc2's operand prologue, gelu' in the epilogue of
    the fc2 input gradient and gelu again in the converter warps of the fc2 weight gradient, so the saved state is x, a
    and the two weights: one hidden-sized tensor instead of autograd's two (fc1 output and gelu output)."""

    @staticmethod
    def forward(ctx, x, W1, b1, W2, b2, approximate):
        x = x.contiguous(); W1 = W1.contiguous(); W2 = W2.contiguous()
        b1 = b1.contiguous() if b1 is not None else None
        b2 = b2.contiguous() if b2 is not None else None
        if x.dim() != 3 or W1.dim() != 2 or W2.dim() != 2 or W1.shape[1] != x.shape[2] or W2.shape[1] != W1.shape[0]:
            raise _lib.HyenaB200Error(f"MlpFn: x (B, L, D), W1 (H, D), W2 (Do, H) expected; got {tuple(x.shape)}, "
                                      f"{tuple(W1.shape)}, {tuple(W2.shape)}")
        a = proj_gemm(x, 0, W1, False, 0, bias=b1)                                  # (B, H, L) = W1 x^T + b1
        y = proj_gemm(a, 1, W2, False, 1, bias=b2, gelu=approximate)                # (B, L, Do) = gelu(a)^T W2^T + b2
        ctx.save_for_backward(x, a, W1, W2)
        ctx.approximate, ctx.has_b1, ctx.has_b2 = approximate, b1 is not None, b2 is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, a, W1, W2 = ctx.saved_tensors
        dy = dy.contiguous()
        _need_cuda(dy)
        approx = ctx.approximate
        need_x, need_w1, need_b1, need_w2, need_b2 = (ctx.needs_input_grad[i] for i in range(5))
        dW2 = proj_wgrad(a, dy, transposed_out=True, gelu=approx) if need_w2 else None    # (Do, H) = sum dy^T gelu(a)
        db2 = dy.sum((0, 1)) if (ctx.has_b2 and need_b2) else None
        dx = dW1 = db1 = None
        if need_x or need_w1 or need_b1:
            da = proj_gemm(dy, 0, W2, True, 0, gelu=approx, gelu_pre=a)                 # (B, H, L) = (dy W2)^T o gelu'(a)
            dx = proj_gemm(da, 1, W1, True, 1) if need_x else None                      # (B, L, D) = da^T W1
            dW1 = proj_wgrad(da, x) if need_w1 else None                                # (H, D) = sum da x
            db1 = da.sum((0, 2)) if (ctx.has_b1 and need_b1) else None
        return dx, dW1, db1, dW2, db2, None


_side_streams = {}


def side_stream(device):
    """A second stream per device for work that is independent of the main chain (weight-gradient GEMMs run there
    while the input-gradient GEMM runs on the caller's stream: one op's cuBLASLt input scan overlaps the other's
    tensor-core phase).  Both GEMMs want the whole chip, so it is OFF unless HYENA_B200_SIDE_STREAM=1."""
    import os
    if os.environ.get("HYENA_B200_SIDE_STREAM", "0") != "1":
        return None
    key = device.index if device.index is not None else torch.cuda.current_device()
    s = _side_streams.get(key)
    if s is None:
        s = torch.cuda.Stream(device=device)
        _side_streams[key] = s
    return s


# ------------------------------------------------------------------------------------------ block glue: add + LayerNorm
_ln_scratch = {}


class AddLayerNormFn(torch.autograd.Function):
    """(y, res_out) = (LayerNorm(x + res) * w + b, x + res) in one pass over HBM (csrc/layernorm.cuh), fp32.

    The pre-norm step of the Block that wraps the mixer (flash-attention/flash_attn/modules/block.py:111-148; with
    fused_dropout_add_ln it is flash_attn.ops.layer_norm.dropout_add_layer_norm(prenorm=True, residual_in_fp32=True),
    dropout p = 0).  ``res`` may be None (first block): res_out is then a copy of x."""

    @staticmethod
    def forward(ctx, x, res, w, b, eps):
        _need_cuda(x, res, w, b)
        if not x.is_contiguous() or (res is not None and (not res.is_contiguous() or res.shape != x.shape)):
            raise _lib.HyenaB200Error("add_layer_norm: x and res must be contiguous and of the same shape")
        D = x.shape[-1]
        if w.numel() != D or (b is not None and b.numel() != D):
            raise _lib.HyenaB200Error(f"add_layer_norm: weight / bias must have {D} elements")
        rows = x.numel() // D
        y = torch.empty_like(x)
        res_out = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        w = w.contiguous()
        b = b.contiguous() if b is not None else None
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().hyena_b200_add_layernorm_fwd(
                _ptr(x), _ptr(res), _ptr(w), _ptr(b), float(eps), _ptr(res_out), _ptr(y),
                _ptr(mean), _ptr(rstd), rows, D, _stream()))
        ctx.save_for_backward(res_out, w, mean, rstd)
        ctx.has_res, ctx.has_b, ctx.D, ctx.rows = res is not None, b is not None, D, rows
        return y, res_out

    @staticmethod
    def backward(ctx, dy, dres):
        r, w, mean, rstd = ctx.saved_tensors
        D, rows = ctx.D, ctx.rows
        dy = dy.contiguous()
        dres = dres.contiguous() if dres is not None else None
        _need_cuda(dy, dres)
        dx = torch.empty_like(r)
        dw = torch.empty(D, dtype=torch.float32, device=r.device)
        db = torch.empty(D, dtype=torch.float32, device=r.device) if ctx.has_b else None
        need = int(_lib.lib().hyena_b200_add_layernorm_scratch_bytes(rows, D))
        key = (r.device.index if r.device.index is not None else torch.cuda.current_device(), _stream())
        sc = _ln_scratch.get(key)
        if sc is None or sc.numel() < need:
            sc = torch.empty(need, dtype=torch.uint8, device=r.device)
            _ln_scratch[key] = sc
        with torch.cuda.device(r.device):
            _lib.check(_lib.lib().hyena_b200_add_layernorm_bwd(
                _ptr(dy), _ptr(dres), _ptr(r), _ptr(w), _ptr(mean), _ptr(rstd), _ptr(dx), _ptr(dw), _ptr(db), rows, D,
                _ptr(sc), sc.numel(), _stream()))
        # the gradient of x and of the incoming residual are the same tensor values
        return dx, (dx if ctx.has_res else None), dw.reshape(w.shape), db, None


def add_layer_norm(x, res, weight, bias, eps):
    return AddLayerNormFn.apply(x, res, weight, bias, eps)


# ------------------------------------------------------------------------------------------ incremental decoding
def decode_hist(p, in_bias, sw, sb, cache):
    """After a prefill of P positions: g_0 = short(v) * short(x_{O-1}) of positions [0, P) into cache.h[0] and the last two
    in_proj outputs (with bias) into cache.tail (csrc/decode.cuh).  p (B, (O+1) D, P) without in_proj.bias."""
    _need_cuda(p, in_bias, sw, sb)
    B, C, P = p.shape
    if not p.is_contiguous() or C != (cache.order + 1) * cache.d_model:
        raise _lib.HyenaB200Error(f"decode_hist: p must be contiguous (B, {(cache.order + 1) * cache.d_model}, P)")
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().hyena_b200_decode_hist(
            _ptr(p), _ptr(in_bias), _ptr(sw), _ptr(sb), _ptr(cache.h), _ptr(cache.tail), B, cache.batch_size,
            cache.d_model, cache.order, P, cache.lcap, _stream()))


def decode_step(p_t, in_bias, sw, sb, cache):
    """One position: y_pre (B, D) of position cache.t from p_t (B, (O+1) D), the in_proj output without its bias.  Runs
    the O-1 recurrences in order, two launches each (csrc/decode.cuh); does not advance cache.t."""
    _need_cuda(p_t, in_bias, sw, sb)
    B = p_t.shape[0]
    D, O = cache.d_model, cache.order
    if not p_t.is_contiguous() or tuple(p_t.shape) != (B, (O + 1) * D):
        raise _lib.HyenaB200Error(f"decode_step: p_t must be contiguous (B, {(O + 1) * D})")
    out = [torch.empty(B, D, dtype=torch.float32, device=p_t.device) for _ in range(O - 1)]
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_step(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part), B, cache.batch_size, D, O,
                o, int(cache.t), cache.lcap, _stream()))
    return out[-1]


# ------------------------------------------------------------------------------------------ windowed steps
# A plain step reads the whole history [0, t).  Inside a window [b, b + Wc) a step reads [b, t) and adds
# F_o[t-b] = sum_{s<b} k_o[t-s] g_o[s], computed for the whole window at once by one FFT convolution of the history
# (the refresh).  HyenaOperator.step opens a window once the cache is long enough and the last WINDOW_AFTER_STEPS operations
# on it were steps: the refresh costs about that many plain steps, so a caller that goes on stepping pays at most about twice
# the cheaper route and one that mixes a few steps with extends pays no refresh.  Derivation from tools/bench_generate.py in
# DESIGN.md section 4.11.
WINDOW = 4096                # positions per window (W)
WINDOW_MIN_T = 1 << 16       # no window below this history: a plain step there is bound by launch latency
WINDOW_AFTER_STEPS = 16      # consecutive steps before a window opens


def decode_window_plan(t, lcap, steps, win_b=0, win_wc=0):
    """Route of a step at position t of a cache with Lcap = lcap whose last ``steps`` operations were steps and whose
    window is [win_b, win_b + win_wc) (win_wc = 0: none): "window" (the window holds t), "refresh" (open the window
    decode_window_bounds(t, lcap) first, then step in it) or "plain"."""
    if win_wc > 0 and win_b <= t < win_b + win_wc:
        return "window"
    if t >= WINDOW_MIN_T and steps >= WINDOW_AFTER_STEPS and t < lcap:
        return "refresh"
    return "plain"


def decode_window_bounds(t, lcap):
    """(b, Wc) of the window a refresh at position t opens: b = t rounded down to a multiple of 4 (history rows stay 16-byte
    aligned), Wc = min(WINDOW, lcap - b)."""
    b = int(t) - int(t) % 4
    return b, min(WINDOW, int(lcap) - b)


def _history_conv(cache, ld, h, o, hist, L):
    """Causal convolution of h[:, :, 0:hist) (zero from hist on) with the first L filter taps of recurrence o -> (B, D, L), on
    the library's filter_spectrum + fftconv_forward with a zero skip term.  h (B, D, >= hist) is g_o by position; ld is the
    row stride of the cache's filter, which is kept reversed, so the filter rows are un-reversed and the history compacted or
    zero-padded first (O(L) copies beside the transforms); h is not read at positions >= hist."""
    D, O = cache.d_model, cache.order
    k = cache.k[:(O - 1) * D * ld].view(D, O - 1, ld)[:, o, ld - L:].flip(-1).contiguous()
    if hist == L:
        u = h[:, :, :L].contiguous()
    else:
        u = torch.zeros(h.shape[0], D, L, dtype=torch.float32, device=h.device)
        u[:, :, :hist] = h[:, :, :hist]
    zero = torch.zeros(D, dtype=torch.float32, device=u.device)
    return fftconv_forward(u, filter_spectrum(k), zero)


def decode_window_refresh(cache):
    """Open the window [b, b + Wc) = decode_window_bounds(cache.t, cache.lcap): per recurrence, F_o = outputs [b, b + Wc) of
    the causal convolution of g_o[0, b) with the first b + Wc filter taps, into cache.win_f (allocated (O-1, B, D, WINDOW)
    on first use).  Reads the history below b only."""
    b, wc = decode_window_bounds(cache.t, cache.lcap)
    if wc < 1:
        raise _lib.HyenaB200Error(f"decode_window_refresh: position {cache.t} leaves no room for a window (Lcap {cache.lcap})")
    O, B, D = cache.order, cache.batch_size, cache.d_model
    if cache.win_f is None or cache.win_f.shape[-1] < wc:
        cache.win_f = None
        cache.win_f = torch.empty(O - 1, B, D, max(WINDOW, wc), dtype=torch.float32, device=cache.h.device)
    for o in range(O - 1):
        cache.win_f[o, :, :, :wc] = _history_conv(cache, cache.h.shape[-1], cache.h[o], o, b, b + wc)[:, :, b:]
    cache.win_b, cache.win_wc = b, wc


def decode_win_step(p_t, in_bias, sw, sb, cache):
    """decode_step at a position cache.t inside the open window: per recurrence the dot product over the window positions
    [b, t) and decode_win_step_kernel, which adds F_o[t-b] (csrc/decode.cuh); does not advance cache.t."""
    _need_cuda(p_t, in_bias, sw, sb)
    B = p_t.shape[0]
    D, O = cache.d_model, cache.order
    if not p_t.is_contiguous() or tuple(p_t.shape) != (B, (O + 1) * D):
        raise _lib.HyenaB200Error(f"decode_win_step: p_t must be contiguous (B, {(O + 1) * D})")
    W = 0 if cache.win_f is None else cache.win_f.shape[-1]
    out = [torch.empty(B, D, dtype=torch.float32, device=p_t.device) for _ in range(O - 1)]
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_win_step(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part),
                0 if cache.win_f is None else _ptr(cache.win_f[o]), B, cache.batch_size, D, O, o, int(cache.t),
                cache.win_b, cache.win_wc, W, cache.lcap, _stream()))
    return out[-1]


def decode_step_auto(p_t, in_bias, sw, sb, cache):
    """One step on the route decode_window_plan selects (refreshing the window first when it says so); counts the step."""
    route = decode_window_plan(cache.t, cache.lcap, cache.steps, cache.win_b, cache.win_wc)
    if route == "refresh":
        decode_window_refresh(cache)
    y = decode_step(p_t, in_bias, sw, sb, cache) if route == "plain" else decode_win_step(p_t, in_bias, sw, sb, cache)
    cache.steps += 1
    return y


# ------------------------------------------------------------------------------------------ extending by n positions
# Direct (decode_ext_dot_kernel) against FFT route (fftconv_forward over the whole t + n history).  The direct kernel reads
# the history and the filter once and does n FMAs per position and channel: memory-bound for small n, then its time grows
# with n; the FFT route costs O((t+n) log(t+n)) whatever n.  tools/bench_extend.py on an H100 (DESIGN.md section 4.10, B = 1,
# D = 256): at t = 2^14, 2^17 and 2^20 the direct route is faster (or even, at 2^20) for n <= 256 and the FFT route for
# n >= 1024, so the threshold sits between them.
EXTEND_FFT_MIN_N = 512


def decode_extend_uses_fft(t, n):
    """True when extending a history of t positions by n runs on the FFT route, False for the direct Toeplitz kernel."""
    return int(n) >= EXTEND_FFT_MIN_N


def _extend_check(p, cache, what):
    _need_cuda(p)
    B, C, n = p.shape if p.dim() == 3 else (0, 0, 0)
    D, O = cache.d_model, cache.order
    if p.dim() != 3 or not p.is_contiguous() or C != (O + 1) * D or n < 1:
        raise _lib.HyenaB200Error(f"{what}: p must be contiguous (B, {(O + 1) * D}, n >= 1); got {tuple(p.shape)}")
    return B, n


def decode_extend_hist(p, in_bias, sw, sb, cache):
    """Short filter of the n positions [cache.t, cache.t + n) from p (B, (O+1) D, n), the in_proj output without its bias,
    carried in from cache.tail -> s (B, (O+1) D, n); writes g_0 of the n positions into cache.h[0] and shifts the tail.  Does
    not advance cache.t."""
    _need_cuda(in_bias, sw, sb)
    B, n = _extend_check(p, cache, "decode_extend_hist")
    s = torch.empty_like(p)
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().hyena_b200_decode_extend_hist(
            _ptr(p), _ptr(in_bias), _ptr(sw), _ptr(sb), _ptr(cache.h), _ptr(cache.tail), _ptr(s), B, cache.batch_size,
            cache.d_model, cache.order, int(cache.t), n, cache.lcap, _stream()))
    return s


def _extend_combine(part, row_stride, j_stride, groups, s, out, o, B, n, cache):
    with torch.cuda.device(s.device):
        _lib.check(_lib.lib().hyena_b200_decode_extend_combine(
            _ptr(part), int(row_stride), int(j_stride), int(groups), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(s), _ptr(out),
            B, cache.batch_size, cache.d_model, cache.order, o, int(cache.t), n, cache.lcap, _stream()))


def _decode_extend(p, in_bias, sw, sb, cache, fft):
    B, n = _extend_check(p, cache, "decode_extend")
    D, O, t = cache.d_model, cache.order, int(cache.t)
    L, ld = t + n, cache.h.shape[-1]
    s = decode_extend_hist(p, in_bias, sw, sb, cache)
    y = torch.empty(B, D, n, dtype=torch.float32, device=p.device)
    if not fft:
        groups = int(_lib.lib().hyena_b200_decode_extend_groups(B, D, t, n))
        part = torch.empty(B, D, n, groups, dtype=torch.float32, device=p.device)
    for o in range(O - 1):
        out = y if o == O - 2 else cache.h[o + 1]
        if fft:
            # recomputes all t + n outputs and keeps the last n
            conv = _history_conv(cache, ld, cache.h[o], o, L, L)
            _extend_combine(conv[:, :, t:], L, 1, 1, s, out, o, B, n, cache)
        else:
            with torch.cuda.device(p.device):
                _lib.check(_lib.lib().hyena_b200_decode_extend_dot(
                    _ptr(cache.h[o]), _ptr(cache.k), _ptr(part), groups, B, cache.batch_size, D, O, o, t, n, cache.lcap,
                    _stream()))
            _extend_combine(part, n * groups, groups, groups, s, out, o, B, n, cache)
    return y


def decode_extend_direct(p, in_bias, sw, sb, cache):
    """y_pre (B, D, n) of the positions [cache.t, cache.t + n) from p (B, (O+1) D, n), the in_proj output without its bias,
    on the direct Toeplitz kernel: per recurrence one decode_ext_dot_kernel over the history and one combine
    (csrc/decode_extend.cuh).  Writes the n positions into the cache's history and tail; does not advance cache.t."""
    return _decode_extend(p, in_bias, sw, sb, cache, fft=False)


def decode_extend_fft(p, in_bias, sw, sb, cache):
    """decode_extend_direct on the FFT route: per recurrence, the causal convolution of the whole history [0, t + n) with
    the first t + n filter taps (filter_spectrum + fftconv_forward), then the same combine kernel."""
    return _decode_extend(p, in_bias, sw, sb, cache, fft=True)


def decode_extend(p, in_bias, sw, sb, cache):
    """decode_extend_direct or decode_extend_fft, as decode_extend_uses_fft(cache.t, n) selects."""
    n = p.shape[-1]
    fn = decode_extend_fft if decode_extend_uses_fft(cache.t, n) else decode_extend_direct
    return fn(p, in_bias, sw, sb, cache)


# ------------------------------------------------------------------------------------------ branched caches (fork)
# Branches of one context share its history tail: with base b <= t0 (a multiple of 4), out_o[t] = F_o[t-b] + the sum over
# the branch's own positions [b, t) + (k_o[0] + bias_o) g_o[t], where F_o[j] = sum_{s<b} k_o[b+j-s] g_o[s] depends on the
# parent row's context only -- the windowed step's identity (section 4.11) with the horizon as the window and a history row per
# branch.  F is computed once per distinct parent row at the fork; no later operation reads the context.  DESIGN.md 4.12.
def decode_branch_bounds(t0, lcap, horizon):
    """(b, Hc, H) of a fork at position t0: b = t0 rounded down to a multiple of 4, Hc = min(horizon rounded up to a multiple
    of 4, lcap - b) positions a branch can hold, H = Hc rounded up to a multiple of 4 (the row stride of its history)."""
    b = int(t0) - int(t0) % 4
    hc = min((int(horizon) + 3) // 4 * 4, int(lcap) - b)
    return b, hc, (hc + 3) // 4 * 4


def _branch_cache(cache, h, tail, f, parent, base, hc):
    """A branched DecodeCache of h.shape[1] rows at cache.t sharing cache's filter; fresh step scratch."""
    R, D, C = h.shape[1], cache.d_model, (cache.order + 1) * cache.d_model
    dev = h.device
    s_t = torch.zeros(R, C, dtype=torch.float32, device=dev)
    part = torch.zeros(R, D, (h.shape[-1] + 1023) // 1024, dtype=torch.float32, device=dev)
    new = type(cache)(cache.owner, R, cache.max_seqlen, cache.lcap, cache.k, cache.bias, h, tail, s_t, part)
    new.t = cache.t
    new._branched, new.base, new.hc, new.f, new.parent = True, base, hc, f, parent
    return new


def decode_fork(cache, rows, horizon):
    """Branches of the unbranched operator cache ``cache`` (host-validated ``rows``, see DecodeCache.fork): F of every
    distinct parent row by one FFT convolution of its history [0, b) per recurrence (_history_conv, as decode_window_refresh
    computes it; none when b = 0), the positions [b, t0) and the tails copied, the device parent index built."""
    t0, O, D = cache.t, cache.order, cache.d_model
    b, hc, H = decode_branch_bounds(t0, cache.lcap, horizon)
    dev = cache.h.device
    uniq = sorted(set(rows))
    slot = {r: i for i, r in enumerate(uniq)}
    f = torch.zeros(O - 1, len(uniq), D, H, dtype=torch.float32, device=dev)
    if b > 0:
        ld = cache.h.shape[-1]
        for o in range(O - 1):
            hist = cache.h[o] if uniq == list(range(cache.batch_size)) else cache.h[o, uniq, :, :b]
            f[o, :, :, :hc] = _history_conv(cache, ld, hist, o, b, b + hc)[:, :, b:]
    ridx = torch.tensor(rows, dtype=torch.long, device=dev)
    h = torch.zeros(O - 1, len(rows), D, H, dtype=torch.float32, device=dev)
    if t0 > b:
        h[:, :, :, :t0 - b] = cache.h[:, ridx, :, b:t0]
    parent = torch.tensor([slot[r] for r in rows], dtype=torch.int32, device=dev)
    return _branch_cache(cache, h, cache.tail.index_select(0, ridx), f, parent, b, hc)


def decode_select(cache, index):
    """The branches ``index`` (host-validated, see DecodeCache.select) of the branched operator cache ``cache``: history,
    tail and parent row copied per row, F shared."""
    idx = torch.tensor(index, dtype=torch.long, device=cache.h.device)
    return _branch_cache(cache, cache.h.index_select(1, idx), cache.tail.index_select(0, idx), cache.f,
                         cache.parent.index_select(0, idx), cache.base, cache.hc)


def _branch_args(cache, B, what):
    if B != cache.batch_size:
        raise _lib.HyenaB200Error(f"{what}: batch size {B} differs from the branched cache's {cache.batch_size}")
    return int(cache.t), cache.base, cache.hc, cache.h.shape[-1]


def decode_branch_step(p_t, in_bias, sw, sb, cache):
    """decode_step on a branched cache: per recurrence the dot product over each branch's positions [b, t) and
    decode_branch_step_kernel, which adds the parent row's F[t-b] (csrc/decode.cuh); does not advance cache.t."""
    _need_cuda(p_t, in_bias, sw, sb)
    B = p_t.shape[0]
    D, O = cache.d_model, cache.order
    if not p_t.is_contiguous() or tuple(p_t.shape) != (B, (O + 1) * D):
        raise _lib.HyenaB200Error(f"decode_branch_step: p_t must be contiguous (B, {(O + 1) * D})")
    t, b, hc, H = _branch_args(cache, B, "decode_branch_step")
    out = [torch.empty(B, D, dtype=torch.float32, device=p_t.device) for _ in range(O - 1)]
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_branch_step(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part), _ptr(cache.f[o]),
                _ptr(cache.parent), B, D, O, o, t, b, hc, H, cache.lcap, _stream()))
    return out[-1]


# ------------------------------------------------------------------------------------------ device-position steps
# The steps above take the position from the host (cache.t), so a captured CUDA graph would replay one position forever.
# These variants read t, the window base and the branch base from cache.pos ([t, win_b, base], int32 on the device) inside
# the kernels, with a grid fixed at capture time to a chunk bound of the route; decode_pos_advance moves t on the device.
# They launch nothing else and allocate nothing but their outputs, so a step built from them can be captured
# (decode.StepGraph).  They sum the same partials in the same order as the host-position kernels: the same bits.
def _dev_step_check(p_t, in_bias, sw, sb, cache, what):
    _need_cuda(p_t, in_bias, sw, sb)
    B = p_t.shape[0]
    D, O = cache.d_model, cache.order
    if not p_t.is_contiguous() or tuple(p_t.shape) != (B, (O + 1) * D):
        raise _lib.HyenaB200Error(f"{what}: p_t must be contiguous (B, {(O + 1) * D})")
    if cache.pos is None:
        raise _lib.HyenaB200Error(f"{what}: the cache has no device position (DecodeCache.sync_position)")
    return B, D, O, [torch.empty(B, D, dtype=torch.float32, device=p_t.device) for _ in range(O - 1)]


def decode_step_dev(p_t, in_bias, sw, sb, cache, t_max):
    """decode_step at the position cache.pos[0] on the device, for positions below t_max (the dot kernel's grid covers
    chunks_for(min(t_max, Lcap)) chunks); does not advance the position."""
    B, D, O, out = _dev_step_check(p_t, in_bias, sw, sb, cache, "decode_step_dev")
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_step_dev(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part), _ptr(cache.pos), B,
                cache.batch_size, D, O, o, int(t_max), cache.lcap, _stream()))
    return out[-1]


def decode_win_step_dev(p_t, in_bias, sw, sb, cache):
    """decode_win_step at the position cache.pos[0] inside the window based at cache.pos[1] on the device (the window
    buffer cache.win_f must be allocated; the host keeps pos[1] and win_f current, see decode_window_refresh)."""
    B, D, O, out = _dev_step_check(p_t, in_bias, sw, sb, cache, "decode_win_step_dev")
    if cache.win_f is None:
        raise _lib.HyenaB200Error("decode_win_step_dev: the cache has no window buffer")
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_win_step_dev(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part), _ptr(cache.win_f[o]),
                _ptr(cache.pos), B, cache.batch_size, D, O, o, cache.win_f.shape[-1], cache.lcap, _stream()))
    return out[-1]


def decode_branch_step_dev(p_t, in_bias, sw, sb, cache):
    """decode_branch_step at the position cache.pos[0] of a branched cache whose base cache.pos[2] is on the device."""
    B, D, O, out = _dev_step_check(p_t, in_bias, sw, sb, cache, "decode_branch_step_dev")
    _branch_args(cache, B, "decode_branch_step_dev")
    with torch.cuda.device(p_t.device):
        for o in range(O - 1):
            first = o == 0
            _lib.check(_lib.lib().hyena_b200_decode_branch_step_dev(
                _ptr(p_t) if first else 0, _ptr(in_bias) if first else 0, _ptr(sw) if first else 0,
                _ptr(sb) if first else 0, _ptr(cache.k), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(cache.tail) if first else 0,
                _ptr(cache.s_t), 0 if first else _ptr(out[o - 1]), _ptr(out[o]), _ptr(cache.part), _ptr(cache.f[o]),
                _ptr(cache.parent), _ptr(cache.pos), B, D, O, o, cache.h.shape[-1], cache.lcap, _stream()))
    return out[-1]


def decode_pos_advance(pos):
    """pos[0] += 1 on the device: the end of a device-position step (once per token for all layers of a stack)."""
    with torch.cuda.device(pos.device):
        _lib.check(_lib.lib().hyena_b200_decode_pos_advance(_ptr(pos), _stream()))


def decode_branch_extend(p, in_bias, sw, sb, cache, fft=None):
    """decode_extend on a branched cache: y_pre (B, D, n) of the positions [t, t + n), t = cache.t, per recurrence over each
    branch's positions [b, t + n) only -- decode_ext_dot_kernel on the branch rows (or, with ``fft``, the FFT convolution of
    them), then decode_branch_combine_kernel, which adds the parent row's F.  ``fft`` None: decode_extend_uses_fft(t - b, n)
    chooses.  Writes the n positions into the branch rows and tails; does not advance cache.t."""
    _need_cuda(in_bias, sw, sb)
    B, n = _extend_check(p, cache, "decode_branch_extend")
    t, b, hc, H = _branch_args(cache, B, "decode_branch_extend")
    D, O, lcap, j = cache.d_model, cache.order, cache.lcap, t - b
    if fft is None:
        fft = decode_extend_uses_fft(j, n)
    lib = _lib.lib()
    s = torch.empty_like(p)
    y = torch.empty(B, D, n, dtype=torch.float32, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(lib.hyena_b200_decode_branch_extend_hist(
            _ptr(p), _ptr(in_bias), _ptr(sw), _ptr(sb), _ptr(cache.h), _ptr(cache.tail), _ptr(s), B, D, O, t, n, b, hc, H,
            lcap, _stream()))
        if not fft:
            groups = int(lib.hyena_b200_decode_extend_groups(B, D, j, n))
            part = torch.empty(B, D, n, groups, dtype=torch.float32, device=p.device)
        for o in range(O - 1):
            out = y if o == O - 2 else cache.h[o + 1]
            if fft:
                conv = _history_conv(cache, (lcap + 3) // 4 * 4, cache.h[o], o, j + n, j + n)
                src, row_stride, j_stride, g = conv[:, :, j:], j + n, 1, 1
            else:
                _lib.check(lib.hyena_b200_decode_branch_extend_dot(
                    _ptr(cache.h[o]), _ptr(cache.k), _ptr(part), groups, B, D, O, o, t, n, b, hc, H, lcap, _stream()))
                src, row_stride, j_stride, g = part, n * groups, groups, groups
            _lib.check(lib.hyena_b200_decode_branch_combine(
                _ptr(src), int(row_stride), int(j_stride), int(g), _ptr(cache.bias), _ptr(cache.h[o]), _ptr(s), _ptr(out),
                _ptr(cache.f[o]), _ptr(cache.parent), B, D, O, o, t, n, b, hc, H, lcap, _stream()))
    return y
