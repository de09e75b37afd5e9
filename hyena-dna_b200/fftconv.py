"""The reference's long-convolution op surface on top of the sm_90a library.

Mirrors /root/reference/src/ops/fftconv.py (``fftconv_func``, ``FFTConvFunc``) and the pybind
module ``fftconv`` it imports (csrc/fftconv/fftconv.cpp:238-241: ``fftconv_fwd`` / ``fftconv_bwd``),
for the fp32, gelu=False, no-dropout, head_dim=1, q=v=None case that HyenaFilter.forward uses
(hyena.py:250-259), plus ``k_rev`` (an anticausal second filter, src/ops/fftconv.py:66-67) and ``fftconv_ref`` with
``bidirectional`` (hyena.py:59-88).  Other options raise.  Works for any L up to 2^20 (the reference stops at 8192).
"""
import torch

from . import ops
from ._lib import HyenaB200Error


def _reject(**flags):
    bad = [k for k, v in flags.items() if v]
    if bad:
        raise HyenaB200Error(f"fftconv options not supported by the sm_90a hot path (no fallback): {bad}")


def _is_packed(filter, H, L):
    return (torch.is_tensor(filter) and filter.dim() == 2 and tuple(filter.shape) == (H, ops.spectrum_elems(L)))


def _filter_to_packed(filter, H, L, fft_size):
    """Accept either the reference's `rfft(k, n=fft_size)` (src/ops/fftconv.py:65; (H, fft_size/2+1) complex64) or the
    packed spectrum from ops.filter_spectrum (H, spectrum_elems(L))."""
    if fft_size and torch.is_tensor(filter) and filter.dim() == 2 and filter.shape == (H, fft_size // 2 + 1) \
            and filter.shape[1] != ops.spectrum_elems(L):
        return ops.spectrum_from_rfft(filter, L, fft_size), True
    if _is_packed(filter, H, L):
        return filter, False
    raise HyenaB200Error(f"fftconv: filter must be rfft(k, n=fft_size) of shape ({H}, fft_size/2+1) or the packed "
                         f"spectrum ({H}, {ops.spectrum_elems(L)}); got {tuple(filter.shape)} with fft_size={fft_size}")


def fftconv_fwd(u, filter, D, v, head_dim, q, dropout_mask, gelu, gelu_inp, gelu_q, fft_size,
                force_fp16_output, output_hbl_layout, fftfp16):
    """Signature and filter convention of csrc/fftconv/fftconv.cpp:53-61: ``filter = torch.fft.rfft(k, n=fft_size)``
    (H, fft_size/2+1) complex64, exactly what src/ops/fftconv.py:65 builds -- converted to the packed spectrum by
    hyena_b200_spectrum_from_rfft.  The packed spectrum from ``ops.filter_spectrum`` is accepted as well.
    fp32 / fp16 / bf16 ``u`` with fp32 math like the reference's dispatch (fftconv.cpp:12-31); L <= 2^20, any parity."""
    _reject(v=v is not None, q=q is not None, head_dim=head_dim != 1, dropout_mask=dropout_mask is not None,
            gelu=gelu, gelu_inp=gelu_inp, gelu_q=gelu_q, output_hbl_layout=output_hbl_layout, fftfp16=fftfp16)
    if u.dim() != 3:
        raise HyenaB200Error("fftconv_fwd: u must be (B, H, L)")
    in_dtype = u.dtype
    if in_dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise HyenaB200Error(f"fftconv_fwd: unsupported input dtype {in_dtype}")
    H, L = u.shape[1], u.shape[2]
    kspec, _ = _filter_to_packed(filter, H, L, fft_size)
    out = ops.fftconv_forward(u.to(torch.float32).contiguous(), kspec, D.reshape(-1).to(torch.float32).contiguous())
    out_dtype = torch.float16 if (force_fp16_output and in_dtype != torch.bfloat16) else in_dtype    # fftconv.cpp:107-110
    return out.to(out_dtype)


def fftconv_bwd(dout, u, filter, D, v, head_dim, q, dropout_mask, gelu, gelu_inp, gelu_q, fft_size,
                output_hbl_layout, fftfp16):
    """Signature of csrc/fftconv/fftconv.cpp:134-143; returns (du, dfilter, dD, dv, dq).  With the reference's natural
    ``filter`` the second output is ``dfilter`` (H, fft_size/2+1) complex64 such that
    ``irfft(dfilter, n=fft_size, norm='forward')[..., :L] == dk`` (fftconv.cpp:235, src/ops/fftconv.py:98); with the
    packed spectrum it is dk (H, L) in the time domain."""
    _reject(v=v is not None, q=q is not None, head_dim=head_dim != 1, dropout_mask=dropout_mask is not None,
            gelu=gelu, gelu_inp=gelu_inp, gelu_q=gelu_q, output_hbl_layout=output_hbl_layout, fftfp16=fftfp16)
    H, L = u.shape[1], u.shape[2]
    kspec, natural = _filter_to_packed(filter, H, L, fft_size)
    du, dk, dD = ops.fftconv_backward(dout.to(torch.float32).contiguous(), u.to(torch.float32).contiguous(), kspec,
                                      D.reshape(-1).to(torch.float32).contiguous())
    du = du.to(u.dtype)
    if natural:
        return du, ops.spectrum_to_rfft(dk, fft_size), dD, None, None
    return du, dk, dD, None, None


def _fftconv_bwd_packed(dout, u, kspec, D):
    du, dk, dD = ops.fftconv_backward(dout.contiguous(), u.contiguous(), kspec, D.contiguous())
    return du, dk, dD, None, None


class FFTConvFunc(torch.autograd.Function):
    """src/ops/fftconv.py:58-103."""

    @staticmethod
    def forward(ctx, u, k, D, dropout_mask=None, gelu=True, force_fp16_output=False, output_hbl_layout=False,
                v=None, head_dim=1, q=None, fftfp16=False, k_rev=None):
        _reject(k_rev=k_rev is not None)          # fftconv_func adds the anticausal half through RevCorrFunc
        if u.dtype != torch.float32 or k.dtype != torch.float32:
            raise HyenaB200Error("fftconv_func: fp32 inputs only")
        if u.dim() != 3:
            raise HyenaB200Error("fftconv_func: u must be (B, H, L)")
        u = u.contiguous()
        H, L = u.shape[1], u.shape[2]
        if k.dim() != 2 or k.shape[0] != H:
            raise HyenaB200Error(f"fftconv_func: k must be (H, Lk) with H = {H}; got {tuple(k.shape)}")
        if D.numel() != H:
            raise HyenaB200Error(f"fftconv_func: D must have H = {H} elements; got {tuple(D.shape)}")
        # rfft(k, n=fft_size) (src/ops/fftconv.py:65) zero-pads a short k and truncates a long one; only k[:, :L]
        # can reach the first L outputs of the causal convolution
        ctx.k_len = k.shape[1]
        if k.shape[1] > L:
            k = k[:, :L]
        elif k.shape[1] < L:
            k = torch.nn.functional.pad(k, (0, L - k.shape[1]))
        D = D.reshape(H).to(torch.float32).contiguous()
        k_f = ops.filter_spectrum(k.contiguous())
        ctx.save_for_backward(u, k_f, D)
        _reject(v=v is not None, q=q is not None, head_dim=head_dim != 1, dropout_mask=dropout_mask is not None,
                gelu=gelu, force_fp16_output=force_fp16_output, output_hbl_layout=output_hbl_layout, fftfp16=fftfp16)
        return ops.fftconv_forward(u, k_f, D)

    @staticmethod
    def backward(ctx, dout):
        u, k_f, D = ctx.saved_tensors
        du, dk, dD, _, _ = _fftconv_bwd_packed(dout, u, k_f, D)
        L = u.shape[2]
        if ctx.k_len > L:
            dk = torch.nn.functional.pad(dk, (0, ctx.k_len - L))
        elif ctx.k_len < L:
            dk = dk[:, :ctx.k_len].contiguous()
        return du, dk, dD, None, None, None, None, None, None, None, None, None


class RevCorrFunc(torch.autograd.Function):
    """y[t] = sum_{s >= t} u[s] k_rev[s - t]: the anticausal half that ``k_f + rfft(k_rev).conj()`` adds to the
    convolution (src/ops/fftconv.py:66-67, hyena.py:63-65).  It is the same correlation the backward pass of the causal
    convolution computes for du, so it runs on the library's backward kernels:
        forward   y      = corr(u, k_rev)                 = fftconv_bwd(dout=u, ., k_rev).du
        backward  du     = causal conv(dy, k_rev)         = fftconv_fwd(dy, k_rev)
                  dk_rev[m] = sum_t u[t] dy[t - m]         = fftconv_bwd(dout=u, u=dy, k_rev).dk"""

    @staticmethod
    def forward(ctx, u, k_rev):
        if u.dtype != torch.float32 or k_rev.dtype != torch.float32 or u.dim() != 3:
            raise HyenaB200Error("k_rev: fp32 u (B, H, L) and k_rev (H, Lk) only")
        u = u.contiguous()
        H, L = u.shape[1], u.shape[2]
        if k_rev.dim() != 2 or k_rev.shape[0] != H:
            raise HyenaB200Error(f"k_rev must be (H, Lk) with H = {H}; got {tuple(k_rev.shape)}")
        ctx.k_len = k_rev.shape[1]
        if k_rev.shape[1] > L:
            k_rev = k_rev[:, :L]
        elif k_rev.shape[1] < L:
            k_rev = torch.nn.functional.pad(k_rev, (0, L - k_rev.shape[1]))
        kspec = ops.filter_spectrum(k_rev.contiguous())
        zero = torch.zeros(H, dtype=torch.float32, device=u.device)
        ctx.save_for_backward(u, kspec, zero)
        return ops.fftconv_backward(u, u, kspec, zero)[0]

    @staticmethod
    def backward(ctx, dy):
        u, kspec, zero = ctx.saved_tensors
        dy = dy.contiguous()
        du = ops.fftconv_forward(dy, kspec, zero)
        dk = ops.fftconv_backward(u, dy, kspec, zero)[1]
        L = u.shape[2]
        if ctx.k_len > L:
            dk = torch.nn.functional.pad(dk, (0, ctx.k_len - L))
        elif ctx.k_len < L:
            dk = dk[:, :ctx.k_len].contiguous()
        return du, dk


def fftconv_func(u, k, D, dropout_mask=None, gelu=True, force_fp16_output=False, output_hbl_layout=False,
                 v=None, head_dim=1, q=None, fftfp16=False, k_rev=None):
    """u (B, H, L), k (H, L), D (H,) -> (B, H, L); src/ops/fftconv.py:105-108.  ``k_rev`` (H, L): second, anticausal
    filter (:66-67)."""
    y = FFTConvFunc.apply(u, k, D, dropout_mask, gelu, force_fp16_output, output_hbl_layout, v, head_dim, q,
                          fftfp16, None)
    if k_rev is not None:
        y = y + RevCorrFunc.apply(u, k_rev)
    return y


def fftconv_ref(u, k, D, dropout_mask=None, gelu=True, k_rev=None, bidirectional=False):
    """Same call as the reference's ``fftconv_ref`` (src/models/sequence/hyena.py:59-88) on the sm_90a kernels.

    ``bidirectional`` there pads the input by ~L/2 on both sides -- to exactly the 2L points of the transform, so nothing is
    left to absorb the wrap-around (:67-73) -- and convolves cyclically with the L-tap filter:
        y[i] = sum_s u[s] kpad[(i - pad_before - s) mod 2L],   pad_before = (L + 2 (L // 2)) // 2 - L // 2.
    That is the causal convolution DELAYED by pad_before samples plus, for the early outputs, the wrapped terms
    sum_m u[i + m] r[m] with r[m] = k[2L - pad_before - m] for L - pad_before < m < L -- a correlation, i.e. the same kernels as
    ``k_rev`` -- plus the un-shifted skip term u * D."""
    _reject(gelu=gelu, dropout_mask=dropout_mask is not None,
            bidirectional_with_k_rev=bidirectional and k_rev is not None)   # (the reference never combines them: hyena.py:261)
    shape = u.shape
    L = shape[-1]
    u3 = u.reshape(-1, shape[-2], L).to(torch.float32)
    k2 = (k[0] if k.dim() == 3 else k).to(torch.float32)
    Dv = D.reshape(-1).to(torch.float32)
    if not bidirectional:
        y = fftconv_func(u3, k2, Dv, gelu=False, k_rev=k_rev)
    else:
        zero = torch.zeros_like(Dv)
        yc = fftconv_func(u3, k2, zero, gelu=False)
        pad_before = (L + 2 * (L // 2)) // 2 - L // 2
        yc = torch.nn.functional.pad(yc[..., :L - pad_before], (pad_before, 0)) if pad_before < L else torch.zeros_like(yc)
        if pad_before > 1:                     # wrapped taps: r[L - pad + 1 .. L - 1] = k[L - 1 .. L - pad + 1]
            r = torch.cat([torch.zeros_like(k2[:, :L - pad_before + 1]), k2[:, L - pad_before + 1:].flip(-1)], dim=1)
            yc = yc + RevCorrFunc.apply(u3.contiguous(), r)
        y = yc + u3 * Dv[None, :, None]
    return y.reshape(shape).to(dtype=u.dtype)
