"""Drop-in HyenaOperator / HyenaFilter backed by the sm_90a library.

Mirrors the public surface of /root/reference/src/models/sequence/hyena.py (same class names,
constructor keywords, state_dict keys and shapes, ``_optim`` attributes, ``filter(L)`` /
``forward`` semantics) for the configuration the HyenaDNA models use -- order=2, num_heads=1,
num_blocks=1, inner_factor=1, activation="id", dropout=0 -- and raises a clear error for options
outside that scope instead of silently diverging.  There is no CPU fallback.
"""
import math

import torch
import torch.nn as nn

from . import ops
from ._lib import HyenaB200Error
from .decode import DecodeCache, StepGraph, _host_index, host_lengths


class OptimModule(nn.Module):
    """register(name, tensor, lr): lr == 0 -> buffer, else Parameter carrying ``_optim`` hyper-parameters
    (src/utils/train.py:142-155)."""

    def register(self, name, tensor, lr=None, wd=0.0):
        if lr == 0.0:
            self.register_buffer(name, tensor)
        else:
            self.register_parameter(name, nn.Parameter(tensor))
            optim = {}
            if lr is not None:
                optim["lr"] = lr
            if wd is not None:
                optim["weight_decay"] = wd
            setattr(getattr(self, name), "_optim", optim)


class Sin(nn.Module):
    """sin(freq * x) with one trainable frequency per feature (hyena.py:96-106).  Kept as a module so
    the state_dict carries ``implicit_filter.{1,3,5}.freq``; evaluated inside the fused filter kernel."""

    def __init__(self, dim, w=10, train_freq=True):
        super().__init__()
        self.freq = nn.Parameter(w * torch.ones(1, dim)) if train_freq else w * torch.ones(1, dim)

    def forward(self, x):
        return torch.sin(self.freq * x)


class PositionalEmbedding(OptimModule):
    """z (1, L, emb_dim) = [t, cos(f w), -sin(f w)], t (1, L, 1) = linspace(0, 1, L)  (hyena.py:109-131)."""

    def __init__(self, emb_dim, seq_len, lr_pos_emb=1e-5, **kwargs):
        super().__init__()
        self.seq_len = seq_len
        t = torch.linspace(0, 1, seq_len)[None, :, None]
        bands = (emb_dim - 1) // 2
        pos = torch.linspace(0, seq_len - 1, seq_len)[None, :, None]
        w = 2 * math.pi * pos / seq_len
        f = torch.linspace(1e-4, bands - 1, bands)[None, None]
        zc = torch.exp(-1j * f * w)
        self.register("z", torch.cat([t, zc.real, zc.imag], dim=-1), lr=lr_pos_emb)
        self.register("t", t, lr=0.0)

    def forward(self, L):
        return self.z[:, :L], self.t[:, :L]


class ExponentialModulation(OptimModule):
    """h * (exp(-t |deltas|) + shift)  (hyena.py:134-155); evaluated inside the fused filter kernel."""

    def __init__(self, d_model, fast_decay_pct=0.3, slow_decay_pct=1.5, target=1e-2, modulation_lr=0.0,
                 shift=0.0, **kwargs):
        super().__init__()
        self.shift = shift
        max_decay = math.log(target) / fast_decay_pct
        min_decay = math.log(target) / slow_decay_pct
        self.register("deltas", torch.linspace(min_decay, max_decay, d_model)[None, None], lr=modulation_lr)

    def forward(self, t, x):
        return x * (torch.exp(-t * self.deltas.abs()) + self.shift)


class HyenaFilter(OptimModule):
    """Implicit long filter (hyena.py:158-267).  ``filter(L)`` -> (1, L, D); ``forward(x, L, k, bias)`` ->
    causal FFT convolution of x (..., D, L) with k plus the bias skip term."""

    def __init__(self, d_model, emb_dim=3, order=16, fused_fft_conv=False, seq_len=1024, lr=1e-3, lr_pos_emb=1e-5,
                 dropout=0.0, w=1, wd=0, bias=True, num_inner_mlps=2, linear_mixer=False, modulate=True,
                 normalized=False, bidirectional=False, **kwargs):
        super().__init__()
        if linear_mixer or num_inner_mlps != 2 or dropout != 0.0:
            raise HyenaB200Error("HyenaFilter: linear_mixer / num_inner_mlps != 2 / "
                                 "dropout are outside the sm_90a hot path (no fallback)")
        if order != 64:
            raise HyenaB200Error(f"HyenaFilter: filter order {order} not supported by the fused kernel (64 only)")
        assert emb_dim % 2 != 0 and emb_dim >= 3, "emb_dim must be odd and greater or equal to 3 (time, sine and cosine)"
        self.d_model, self.emb_dim, self.seq_len, self.modulate = d_model, emb_dim, seq_len, modulate
        self.use_bias = bias
        self.fused_fft_conv = fused_fft_conv      # accepted for config compatibility; the fused path is always on
        self.bias = nn.Parameter(torch.randn(d_model))
        self.dropout = nn.Dropout(dropout)
        self.bidirectional = bidirectional
        self.normalized = normalized

        act = Sin(dim=order, w=w)
        self.pos_emb = PositionalEmbedding(emb_dim, seq_len, lr_pos_emb)
        self.implicit_filter = nn.Sequential(nn.Linear(emb_dim, order), act)
        for _ in range(num_inner_mlps):
            self.implicit_filter.append(nn.Linear(order, order))
            self.implicit_filter.append(act)
        self.implicit_filter.append(nn.Linear(order, d_model, bias=False))
        self.modulation = ExponentialModulation(d_model, **kwargs)
        for c in self.implicit_filter.children():
            for name, _ in c.state_dict().items():
                setattr(getattr(c, name), "_optim", {"weight_decay": wd, "lr": lr})

    def filter_channel_major(self, L):
        """k (D, L): the layout the convolution kernels consume.

        With ``self.cache_filter`` set (see stack.CheckpointedHyenaStack) the generated filter is kept and reused while
        none of the tensors it depends on has changed (torch's per-tensor version counters: an optimizer step or any
        in-place write invalidates it).  Under activation checkpointing every layer's forward runs twice per step
        (long_conv_lm.py:39-45,196-199): the recompute then skips the filter kernels -- at batch 1 they are a third of
        the custom-kernel time of a forward."""
        f = self.implicit_filter
        args = (self.pos_emb.z, self.pos_emb.t, f[0].weight, f[0].bias, f[2].weight, f[2].bias, f[4].weight, f[4].bias,
                f[6].weight, f[1].freq, self.modulation.deltas)
        cached = None
        if getattr(self, "cache_filter", False):
            key = (int(L), float(self.modulation.shift), bool(self.modulate)) + tuple((a.data_ptr(), a._version) for a in args)
            c = getattr(self, "_filter_cache", None)
            if c is not None and c[0] == key:
                cached = c[1]
        k = ops.HyenaFilterFn.apply(*args, float(self.modulation.shift), bool(self.modulate), int(L), cached)
        if getattr(self, "cache_filter", False) and cached is None:
            self._filter_cache = (key, k.detach())
        if self.normalized:                     # hyena.py:235-236: L1 norm over the channels of every position
            k = ops.FilterL1NormFn.apply(k)
        return k

    def filter(self, L, *args, **kwargs):
        return self.filter_channel_major(L).transpose(0, 1).unsqueeze(0)

    def forward(self, x, L, k=None, bias=None, *args, **kwargs):
        from .fftconv import fftconv_func, fftconv_ref
        if self.bidirectional:                 # hyena.py:261: fftconv_ref(..., bidirectional=self.bidirectional)
            if k is None:
                k = self.filter_channel_major(L)
            else:
                k = k[0] if type(k) is tuple else k
                if k.dim() == 3:
                    k = k[0].transpose(0, 1)
            b = self.bias if bias is None else bias
            b = b if self.use_bias else 0 * b
            if x.dim() == 5:
                bb, h, v, zz, l = x.shape
                x3 = x.permute(0, 3, 1, 2, 4).reshape(bb * zz, h * v, l)
                y = fftconv_ref(x3, k, b.reshape(-1), None, gelu=False, bidirectional=True)
                return y.reshape(bb, zz, h, v, l).permute(0, 2, 3, 1, 4).to(dtype=x.dtype)
            return fftconv_ref(x, k, b.reshape(-1), None, gelu=False, bidirectional=True)
        if k is None:
            k = self.filter_channel_major(L)
        else:
            k = k[0] if type(k) is tuple else k
            if k.dim() == 3:
                k = k[0].transpose(0, 1)
        if bias is None:
            bias = self.bias
        bias = bias if self.use_bias else 0 * bias
        bias = bias.reshape(-1).to(torch.float32)
        if x.dim() == 5:        # the reference operator's layout (b, heads, v, blocks, l)  (hyena.py:396-402, :423)
            b, h, v, z, l = x.shape
            x3 = x.permute(0, 3, 1, 2, 4).reshape(b * z, h * v, l)
            y = fftconv_func(x3.to(torch.float32), k, bias, gelu=False)
            return y.reshape(b, z, h, v, l).permute(0, 2, 3, 1, 4).to(dtype=x.dtype)
        shape = x.shape
        y = fftconv_func(x.reshape(-1, shape[-2], shape[-1]).to(torch.float32), k, bias, gelu=False)
        return y.reshape(shape).to(dtype=x.dtype)


class _InProj(torch.autograd.Function):
    """p = W u^T written channel-major (B, 3D, L) straight from the GEMM: no transpose pass
    (replaces hyena.py:391-392).  The bias is added inside the fused kernels."""

    @staticmethod
    def forward(ctx, u, W):
        u = u.contiguous(); W = W.contiguous()
        ctx.save_for_backward(u, W)
        B, L, D = u.shape
        C3 = W.shape[0]
        mode = ops.proj_mode()
        if mode == "tc":
            return ops.proj_gemm(u, 0, W, False, 0)                       # p (B, 3D, L) = W u^T, channel-major
        if mode == "torch":
            return torch.bmm(W.unsqueeze(0).expand(B, -1, -1), u.transpose(1, 2))
        p = torch.empty(B, C3, L, dtype=torch.float32, device=u.device)
        # col-major: P^T (L x 3D, ld L) = U (L x D) W^T (D x 3D);  U stored (D x L, ld D) -> op T
        ops.gemm(1, 0, L, C3, D, u, D, L * D, W, D, 0, p, L, C3 * L, batch=B)
        return p

    @staticmethod
    def backward(ctx, dp):
        u, W = ctx.saved_tensors
        B, L, D = u.shape
        C3 = W.shape[0]
        dp = dp.contiguous()
        mode = ops.proj_mode()
        if mode == "tc":
            du = ops.proj_gemm(dp, 1, W, True, 1) if ctx.needs_input_grad[0] else None      # du = dp^T W
            dW = ops.proj_wgrad(dp, u) if ctx.needs_input_grad[1] else None                 # dW = sum dp u
            return du, dW
        if mode == "torch":
            du = torch.matmul(dp.transpose(1, 2), W) if ctx.needs_input_grad[0] else None
            dW = torch.bmm(dp, u).sum(0) if ctx.needs_input_grad[1] else None
            return du, dW
        du = dW = None
        if ctx.needs_input_grad[1]:
            dW = torch.empty_like(W)
            # dW^T (D x 3D, ld D) = sum_b U_b^T (D x L, stored, op N) dP_b^T (L x 3D, stored ld L, op N)
            for b in range(B):
                ops.gemm(0, 0, D, C3, L, u[b], D, 0, dp[b], L, 0, dW, D, 0, batch=1, beta=0.0 if b == 0 else 1.0)
        if ctx.needs_input_grad[0]:
            du = torch.empty_like(u)
            # dU^T (D x L, ld D) = W^T (D x 3D, stored ld D, op N) dP (3D x L; stored (L x 3D, ld L) -> op T)
            ops.gemm(0, 1, D, L, C3, W, D, 0, dp, L, C3 * L, du, D, L * D, batch=B)
        return du, dW


class _OutProj(torch.autograd.Function):
    """y = y_pre^T W^T + b consuming channel-major y_pre (B, D, L) (replaces hyena.py:432-440)."""

    @staticmethod
    def forward(ctx, y_pre, W, b):
        y_pre = y_pre.contiguous(); W = W.contiguous()
        ctx.save_for_backward(y_pre, W)
        ctx.has_bias = b is not None
        B, C, L = y_pre.shape
        Do = W.shape[0]
        mode = ops.proj_mode()
        if mode == "tc":
            return ops.proj_gemm(y_pre, 1, W, False, 1, bias=b.contiguous() if b is not None else None)
        if mode == "torch":
            y = torch.bmm(y_pre.transpose(1, 2), W.t().unsqueeze(0).expand(B, -1, -1))
            if b is not None:
                y += b
            return y
        y = torch.empty(B, L, Do, dtype=torch.float32, device=y_pre.device)
        # Y^T (Do x L, ld Do) = W (Do x C; stored (C x Do, ld C) -> op T) Ypre (C x L; stored (L x C, ld L) -> op T)
        ops.gemm(1, 1, Do, L, C, W, C, 0, y_pre, L, C * L, y, Do, L * Do, batch=B,
                 bias=b.contiguous() if b is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        y_pre, W = ctx.saved_tensors
        B, C, L = y_pre.shape
        Do = W.shape[0]
        dy = dy.contiguous()
        mode = ops.proj_mode()
        if mode == "tc":
            d_pre = ops.proj_gemm(dy, 0, W, True, 0) if ctx.needs_input_grad[0] else None          # (B, C, L) = W^T dy^T
            dW = ops.proj_wgrad(y_pre, dy, transposed_out=True) if ctx.needs_input_grad[1] else None   # (Do, C)
            db = dy.sum((0, 1)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
            return d_pre, dW, db
        if mode == "torch":
            d_pre = torch.bmm(W.t().unsqueeze(0).expand(B, -1, -1), dy.transpose(1, 2)) if ctx.needs_input_grad[0] else None
            dW = torch.bmm(dy.transpose(1, 2), y_pre.transpose(1, 2)).sum(0) if ctx.needs_input_grad[1] else None
            db = dy.sum((0, 1)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
            return d_pre, dW, db
        d_pre = dW = db = None
        if ctx.needs_input_grad[1]:
            dW = torch.empty_like(W)
            # dW^T (C x Do, ld C) = sum_b Ypre_b (C x L; stored (L x C, ld L) -> op T) dY_b (L x Do; stored (Do x L) -> op T)
            for b in range(B):
                ops.gemm(1, 1, C, Do, L, y_pre[b], L, 0, dy[b], Do, 0, dW, C, 0, batch=1, beta=0.0 if b == 0 else 1.0)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum((0, 1))
        if ctx.needs_input_grad[0]:
            d_pre = torch.empty_like(y_pre)
            # dYpre^T (L x C, ld L) = dY (L x Do; stored (Do x L, ld Do) -> op T) W (Do x C; stored (C x Do, ld C) -> op T)
            ops.gemm(1, 1, L, C, Do, dy, Do, L * Do, W, C, 0, d_pre, L, C * L, batch=B)
        return d_pre, dW, db


class LeftPadding:
    """A validated left-padding mask (HyenaOperator.check_mask): the rows' first real positions on the host (``starts``)
    and on the mask's device or u's device (``row_start``, (B,) int32).  Block and Backbone pass it on to their mixers so
    that a mask is validated, and copied, once per call."""

    def __init__(self, starts, row_start, positions):
        self.starts, self.row_start, self.positions = starts, row_start, positions


def host_mask_starts(mask, batch, positions, device):
    """mask (batch, positions), bool or integer 0/1, on the CPU or on ``device`` -> LeftPadding, checked with one
    device-to-host copy of per-row results for a device mask.  Row b must be zeros followed by at least one one (the
    attention mask of a left-padded batch); its real tokens are its last mask[b].sum() positions."""
    if isinstance(mask, LeftPadding):
        if len(mask.starts) != batch or mask.positions != positions or mask.row_start.device != device:
            raise HyenaB200Error("this LeftPadding was validated for another input shape or device")
        return mask
    if not torch.is_tensor(mask):
        raise HyenaB200Error(f"mask must be a ({batch}, {positions}) bool or integer tensor; got {type(mask).__name__}")
    if mask.dtype.is_floating_point or mask.dtype.is_complex:
        raise HyenaB200Error(f"mask must be bool or integer 0/1; got {mask.dtype}")
    if tuple(mask.shape) != (batch, positions):
        raise HyenaB200Error(f"mask must be ({batch}, {positions}) like the input's (B, L); got {tuple(mask.shape)}")
    if mask.device.type != "cpu" and mask.device != device:
        raise HyenaB200Error(f"mask must be on the CPU or on the input's device {device}; got {mask.device}")
    m = mask.detach()
    badval = ((m != 0) & (m != 1)).any(1) if m.dtype != torch.bool else torch.zeros_like(m[:, 0])
    m = m != 0
    n = m.sum(1)
    unordered = (m[:, :-1] & ~m[:, 1:]).any(1)                 # a one followed by a zero
    info = torch.stack([n, badval.to(n.dtype), unordered.to(n.dtype)]).cpu().tolist()
    for b in range(batch):
        if info[1][b]:
            raise HyenaB200Error(f"mask values must be 0 or 1 (row {b})")
    for b in range(batch):
        if info[0][b] == 0:
            raise HyenaB200Error(f"mask row {b} is empty: every row needs at least one real token")
        if info[2][b]:
            raise HyenaB200Error(f"mask row {b} is not left-padded: a row must be zeros (pads) followed by ones "
                                 "(real tokens)")
    starts = [positions - k for k in info[0]]
    row_start = (positions - n).to(torch.int32)
    if row_start.device != device and device.type == "cuda":
        row_start = row_start.pin_memory().to(device, non_blocking=True)
    return LeftPadding(starts, row_start, positions)


class Packing:
    """Validated packed sequences (HyenaOperator.check_packed): ``cu`` the cumulative lengths on the host, ``plan`` the
    bucket plan (ops.packed_plan), ``tables`` its row bases and starts on the device, ``max_len`` the longest sequence.
    Block and Backbone pass it on to their mixers as ``cu_seqlens`` so that it is validated, and copied, once per call."""

    def __init__(self, cu, plan, tables, max_len, device):
        self.cu, self.plan, self.tables, self.max_len, self.device = cu, plan, tables, max_len, device

    @property
    def total(self):
        return self.cu[-1]


def host_cu_seqlens(cu_seqlens, total, device):
    """cu_seqlens ((N+1,) integer, on the CPU or on ``device``) -> the list on the host, checked with one device-to-host
    copy: cu[0] == 0, non-decreasing, cu[N] == total."""
    if not torch.is_tensor(cu_seqlens):
        raise HyenaB200Error(f"cu_seqlens must be a (N+1,) integer tensor; got {type(cu_seqlens).__name__}")
    if cu_seqlens.dtype.is_floating_point or cu_seqlens.dtype.is_complex or cu_seqlens.dtype == torch.bool:
        raise HyenaB200Error(f"cu_seqlens must be an integer tensor; got {cu_seqlens.dtype}")
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2:
        raise HyenaB200Error(f"cu_seqlens must be (N+1,) with N >= 1; got shape {tuple(cu_seqlens.shape)}")
    if cu_seqlens.device.type != "cpu" and cu_seqlens.device != device:
        raise HyenaB200Error(f"cu_seqlens must be on the CPU or on the input's device {device}; got {cu_seqlens.device}")
    cu = [int(x) for x in cu_seqlens.detach().cpu().tolist()]
    if cu[0] != 0:
        raise HyenaB200Error(f"cu_seqlens[0] must be 0; got {cu[0]}")
    for i in range(len(cu) - 1):
        if cu[i + 1] < cu[i]:
            raise HyenaB200Error(f"cu_seqlens must be non-decreasing; cu_seqlens[{i + 1}] = {cu[i + 1]} < {cu[i]}")
    if cu[-1] != total:
        raise HyenaB200Error(f"cu_seqlens[-1] = {cu[-1]} must equal the number of packed positions {total}")
    return cu


class HyenaOperator(nn.Module):
    """Hyena operator (hyena.py:270-448): order 2 as one fused pass on sm_90a, order >= 3 as a chain of its kernels.

    forward(u: (B, L, D)) -> (B, L, D) (or ``(y, None)`` when return_state).  Unknown keyword arguments
    (layer_idx, device, dtype, ...) fall through to the filter exactly as in the reference."""

    def __init__(self, d_model, l_max, order=2, filter_order=64, num_heads=1, inner_factor=1, num_blocks=1,
                 fused_bias_fc=False, outer_mixing=False, dropout=0.0, filter_dropout=0.0, filter_cls="hyena-filter",
                 post_order_ffn=False, jit_filter=False, short_filter_order=3, activation="id", return_state=False,
                 **filter_args):
        super().__init__()
        unsupported = {"order": order < 2, "num_heads": num_heads != 1, "inner_factor": inner_factor != 1,
                       "num_blocks": num_blocks != 1, "outer_mixing": outer_mixing, "dropout": dropout != 0.0,
                       "filter_dropout": filter_dropout != 0.0, "post_order_ffn": post_order_ffn,
                       "jit_filter": jit_filter, "short_filter_order": short_filter_order != 3,
                       "activation": activation not in ("id", "identity", None),
                       "filter_cls": filter_cls != "hyena-filter", "fused_bias_fc": fused_bias_fc}
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise HyenaB200Error(f"HyenaOperator options outside the sm_90a hot path (no fallback): {bad}")
        self.d_model, self.l_max, self.order = d_model, l_max, order
        self.num_heads, self.inner_factor, self.num_blocks = num_heads, inner_factor, num_blocks
        self.block_dim, self.head_dim = l_max // num_blocks, d_model // num_heads
        self.filter_order, self.short_filter_order = filter_order, short_filter_order
        self.post_order_ffn, self.jit_filter, self.outer_mixing = post_order_ffn, jit_filter, outer_mixing
        self.filter_dropout, self.return_state = filter_dropout, return_state
        self.activation = nn.Identity()
        self.dropout = nn.Dropout(dropout)
        self.out_proj = nn.Linear(d_model * inner_factor, d_model)
        self.in_proj = nn.Linear(d_model, (order + 1) * d_model)
        total_width = d_model * inner_factor * (order + 1)
        self.short_filter = nn.Conv1d(total_width, total_width, short_filter_order, groups=total_width,
                                      padding=short_filter_order - 1)
        filter_args.pop("channels", None)
        self.filter_fn = HyenaFilter(self.head_dim * inner_factor * (order - 1), order=filter_order, seq_len=l_max,
                                     channels=1, dropout=filter_dropout, **filter_args)

    def forward(self, u, *args, lengths=None, mask=None, cu_seqlens=None, max_seqlen=None, stream=False, **kwargs):
        """``lengths`` (B integers in [1, L]): u is left-padded, row b's real tokens are its last lengths[b] positions.  Its
        outputs there do not depend on the padding: they are the outputs of the unpadded row (DESIGN.md section 4.14); at a
        pad position the output is out_proj(0) = out_proj.bias.  Inference only: with grad required it raises (use
        ``mask``, or train on right-padded batches, where a causal operator is exact as it stands).

        ``mask`` ((B, L) bool or integer 0/1, the attention mask of a left-padded batch, on the CPU or on u's device): the
        same masked operator, differentiable (DESIGN.md section 4.17).  Outputs and every gradient at real positions are
        the unpadded rows', parameter gradients are the sums over rows of the unpadded rows', du is 0 at the pads and the
        pad contents (NaN and inf included) change nothing.  Under torch.no_grad() it gives the bits of
        ``forward(u, lengths=mask.sum(-1))``.  Not with ``lengths`` or a DecodeCache (decoding takes ``lengths``).

        ``cu_seqlens`` ((N+1,) integer cumulative lengths, on the CPU or on u's device; flash-attention's unpadded
        convention): u is (total, D) or (1, total, D), sequences packed without padding, sequence i at positions
        [cu_seqlens[i], cu_seqlens[i+1]).  Each sequence runs as if alone (DESIGN.md section 4.18); the output has u's
        shape.  ``max_seqlen``, when given, must be at least the longest sequence.  Order 2 with a causal filter only;
        not with ``lengths``, ``mask`` or a DecodeCache.

        ``stream=True``: u (B, L, D) of any length, every position's output (DESIGN.md section 4.21).  The output at t is
        the layer with its l_max-tap causal convolution applied as a stream, the outputs an unbounded DecodeCache gives,
        computed on overlapping windows of the FFT core; for L <= l_max it is ``forward(u)``, bit for bit.  Inference
        only (run under torch.no_grad()), a causal filter, l_max <= 2^20 - 2; not with ``lengths``, ``mask``,
        ``cu_seqlens`` or a DecodeCache."""
        cache = kwargs.get("inference_params")
        if stream:
            plan = self.check_stream(u, cache, lengths, mask, cu_seqlens)
            if plan is not None:
                y = self._forward_stream(u, plan)
                return (y, None) if self.return_state else y
        if cu_seqlens is not None:
            y = self._forward_packed(u, self.check_packed(u, cu_seqlens, max_seqlen, cache, lengths, mask))
            return (y, None) if self.return_state else y
        if mask is not None:
            y = self._forward_masked(u, self.check_mask(u, mask, cache, lengths))
            return (y, None) if self.return_state else y
        if isinstance(cache, DecodeCache):
            # incremental decoding driven by the caller's model (LMBackbone passes inference_params to every mixer,
            # long_conv_lm.py:375-376); any other inference_params object is ignored, as the reference does
            # a fresh cache takes several positions as a prefill, one position is a step, several positions on a cache
            # that already holds history extend it
            c = cache.for_module(self)
            n = u.shape[-2]
            if lengths is not None:
                y = self.prefill(u, c, lengths) if c.t == 0 and not c.branched else \
                    self.step(u, c, lengths) if n == 1 else self.extend(u, c, lengths)
            else:
                y = self.prefill(u, c) if (c.t == 0 and n > 1) else self.step(u, c) if n == 1 else self.extend(u, c)
            return (y, None) if self.return_state else y
        if lengths is not None:
            y = self._forward_left_padded(u, lengths)
            return (y, None) if self.return_state else y
        if not u.is_cuda:
            raise HyenaB200Error("HyenaOperator (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        in_dtype = u.dtype
        u = u.to(torch.float32)
        l = u.size(-2)
        l_filter = min(l, self.l_max)
        k = self.filter_fn.filter_channel_major(l_filter)                           # (D*(order-1), l_filter)
        fb = self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias
        kspec = None
        if self.order == 2 and getattr(self.filter_fn, "cache_filter", False):
            # spectrum of the cached filter, kept with it (same invalidation: it is keyed on the cached k tensor)
            c = getattr(self, "_kspec_cache", None)
            kkey = (k.data_ptr(), k._version, tuple(k.shape))
            if c is not None and c[0] == kkey:
                kspec = c[1]
            else:
                kspec = ops.filter_spectrum(k.detach())
                self._kspec_cache = (kkey, kspec)
        if self.order > 2 or self.filter_fn.bidirectional:
            y_pre = self._forward_chained(u, k, fb, l_filter)
        elif ops.proj_mode() == "tc" and l_filter == l:
            # one autograd node: in_proj GEMM + fused core; backward feeds ds straight into the projection GEMMs
            y_pre = ops.HyenaInCoreFn.apply(u, self.in_proj.weight, self.in_proj.bias, self.short_filter.weight,
                                            self.short_filter.bias, k, fb, kspec)
        else:
            p = _InProj.apply(u, self.in_proj.weight)                               # (B, 3D, l)
            if l_filter < l:
                p = p[..., :l_filter].contiguous()
            y_pre = ops.HyenaCoreFn.apply(p, self.in_proj.bias, self.short_filter.weight, self.short_filter.bias, k, fb,
                                          kspec)
        y = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias).to(in_dtype)
        if self.return_state:
            return y, None
        return y

    def check_stream(self, u, cache=None, lengths=None, mask=None, cu_seqlens=None, device=True):
        """Every host check of ``forward(u, stream=True)`` without device work (Block and Backbone run it before their first
        kernel) -> the plan (ops.stream_plan), or None when L <= l_max (then ``forward(u)`` runs).  ``device`` False: all
        but the check that u is on the GPU (a Backbone checks every layer before it checks the device)."""
        if lengths is not None or mask is not None or cu_seqlens is not None:
            raise HyenaB200Error("stream=True does not combine with lengths, mask or cu_seqlens: a streamed row is one "
                                 "sequence from its first position")
        if isinstance(cache, DecodeCache):
            raise HyenaB200Error("stream=True does not combine with a DecodeCache: decode with prefill, step and extend")
        if self.filter_fn.bidirectional:
            raise HyenaB200Error("stream=True needs a causal filter; this HyenaFilter is bidirectional")
        if torch.is_grad_enabled() and (u.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise HyenaB200Error("forward(u, stream=True) is inference only (run under torch.no_grad())")
        if u.dim() != 3 or u.shape[-1] != self.d_model or u.shape[1] < 1:
            raise HyenaB200Error(f"stream=True takes u (B, L, {self.d_model}) with L >= 1; got {tuple(u.shape)}")
        if self.l_max > ops.STREAM_MAX_WINDOW - 2:
            raise HyenaB200Error(f"stream=True: l_max = {self.l_max} leaves no room for an output in a window of at "
                                 f"most {ops.STREAM_MAX_WINDOW} positions (l_max <= {ops.STREAM_MAX_WINDOW - 2})")
        if device and not u.is_cuda:
            raise HyenaB200Error("HyenaOperator (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        B, L = u.shape[0], u.shape[1]
        return None if L <= self.l_max else ops.stream_plan(L, self.l_max, self.order, B)

    def _forward_stream(self, u, plan):
        """forward(u, stream=True) past l_max: the chunks of ``plan`` in turn.  A chunk takes every row's positions
        [in_start, out_end) as one packed (1, B n) in_proj GEMM, the core on the chunk's overlapping windows (order 2:
        hyena_b200_core_fwd_windows; order >= 3: the short filter and gates in torch, every recurrence's convolution as
        its own windowed pass, hyena_b200_fftconv_fwd_windows), out_proj, and keeps the outputs [out_start, out_end)."""
        B, L, D = u.shape
        dev, L_b = u.device, plan.L_b
        y = torch.empty(B, L, D, dtype=u.dtype, device=dev)
        with torch.no_grad():
            k = self.filter_fn.filter_channel_major(self.l_max)                      # (D*(order-1), l_max)
            fb = (self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias).reshape(-1)
            fb = fb.to(torch.float32).contiguous()
            C = self.short_filter.weight.shape[0]
            sw = self.short_filter.weight.reshape(C, -1).contiguous()
            sb = self.short_filter.bias.contiguous()
            ib = self.in_proj.bias.contiguous() if self.in_proj.bias is not None else None
            O1 = self.order - 1
            kk = k.reshape(D, O1, self.l_max)                                        # filter channels are ordered (v o)
            kspecs = [ops.filter_spectrum(ops._bucket_filter(kk[:, o].contiguous(), L_b)) for o in range(O1)]
            bb = fb.reshape(D, O1)
            tables = {}
            for s, a, e in plan.chunks:
                n = e - s
                if n not in tables:
                    tables[n] = ops.stream_tables(plan.windows(n), B, n if self.order == 2 else D * n, dev)
                uc = u[:, s:e].to(torch.float32)
                if self.order == 2:
                    # one packed (1, B n) layout: row b's position t at b n + t, padded to a multiple of 4 positions
                    total = B * n
                    tp = -(-total // 4) * 4
                    u32 = uc.reshape(total, D)
                    if tp != total:
                        u32 = torch.nn.functional.pad(u32, (0, 0, 0, tp - total))
                    p = _InProj.apply(u32[None].contiguous(), self.in_proj.weight)    # (1, 3D, tp)
                    y_pre = ops.core_forward_windows(p, ib, sw, sb, kspecs[0], fb, L_b, tables[n], total)
                    yc = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias)[0, :total].reshape(B, n, D)
                else:
                    y_pre = self._stream_chained(uc.contiguous(), kspecs, bb, L_b, tables[n])
                    yc = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias)
                y[:, a:e] = yc[:, a - s:]
        return y

    def _stream_chained(self, u, kspecs, bb, L_b, tables):
        """y_pre (B, D, n) of order >= 3 on a chunk u (B, n, D): _forward_chained's recurrence with every convolution a
        windowed pass over the chunk's rows (ops.fftconv_forward_windows, channel stride n)."""
        D = self.d_model
        n = u.shape[1]
        p = _InProj.apply(u, self.in_proj.weight)                                   # (B, (order+1) D, n)
        if self.in_proj.bias is not None:
            p = p + self.in_proj.bias[None, :, None]
        uc = torch.nn.functional.conv1d(p, self.short_filter.weight, self.short_filter.bias,
                                        padding=self.short_filter_order - 1, groups=p.shape[1])[..., :n]
        *x, v = uc.split(D, dim=1)
        for o, x_i in enumerate(reversed(x[1:])):
            v = ops.fftconv_forward_windows((v * x_i).contiguous(), kspecs[o], bb[:, o].contiguous(), L_b, tables)
        return (v * x[0]).contiguous()

    def _padded_checks(self, u, what, hint=""):
        """Host validation of a left-padded input's filter and shape -> (B, P); ``hint`` ends a too-long input's error."""
        if self.filter_fn.bidirectional:
            raise HyenaB200Error(f"{what} needs a causal filter; this HyenaFilter is bidirectional")
        if u.dim() != 3 or u.shape[-1] != self.d_model:
            raise HyenaB200Error(f"left-padded input must be (B, L, {self.d_model}); got {tuple(u.shape)}")
        B, P = u.shape[0], u.shape[1]
        if P > self.l_max:
            raise HyenaB200Error(f"left-padded input of {P} positions exceeds l_max = {self.l_max}{hint}")
        return B, P

    def _ragged_checks(self, u, lengths, hint=""):
        """Host validation of a left-padded input before any device work -> the rows' first real positions."""
        B, P = self._padded_checks(u, "lengths", hint)
        return [P - n for n in host_lengths(lengths, B, P)]

    def check_mask(self, u, mask, cache=None, lengths=None):
        """Every host check of ``forward(u, mask=mask)`` without device work (Block and Backbone run it before their first
        kernel) -> LeftPadding (``mask`` may be one already)."""
        if lengths is not None:
            raise HyenaB200Error("pass mask or lengths, not both: they describe the same left padding")
        if isinstance(cache, DecodeCache):
            raise HyenaB200Error("mask does not combine with a DecodeCache: decoding takes lengths= (a left-padded prefill)")
        B, P = self._padded_checks(u, "mask")
        pad = host_mask_starts(mask, B, P, u.device)
        if not u.is_cuda:
            raise HyenaB200Error("HyenaOperator (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        return pad

    def check_packed(self, u, cu_seqlens, max_seqlen=None, cache=None, lengths=None, mask=None):
        """Every host check of ``forward(u, cu_seqlens=..., max_seqlen=...)`` without device work (Block and Backbone
        run it before their first kernel) -> Packing (``cu_seqlens`` may be one already)."""
        if lengths is not None or mask is not None:
            raise HyenaB200Error("cu_seqlens does not combine with lengths or mask: packed sequences have no padding")
        if isinstance(cache, DecodeCache):
            raise HyenaB200Error("forward(u, cu_seqlens=...) does not combine with a DecodeCache: packed prompts enter a "
                                 "cache through prefill(u, cache, cu_seqlens=...) or admit(u, cache, rows, cu_seqlens=...)")
        return self._packed_on_device(u, self._packed_host(u, cu_seqlens, max_seqlen))

    def _packed_host(self, u, cu_seqlens, max_seqlen, hint=""):
        """The host checks of packed input that need no device -> Packing without its plan (or the given Packing);
        ``hint`` ends a too-long sequence's error."""
        if self.order != 2:
            raise HyenaB200Error(f"cu_seqlens needs order 2; this operator has order {self.order}")
        if self.filter_fn.bidirectional:
            raise HyenaB200Error("cu_seqlens needs a causal filter; this HyenaFilter is bidirectional")
        if not (u.dim() == 2 or (u.dim() == 3 and u.shape[0] == 1)) or u.shape[-1] != self.d_model:
            raise HyenaB200Error(f"packed input must be (total, {self.d_model}) or (1, total, {self.d_model}); "
                                 f"got {tuple(u.shape)}")
        total = u.shape[-2]
        if isinstance(cu_seqlens, Packing):
            if cu_seqlens.total != total or cu_seqlens.device != u.device:
                raise HyenaB200Error("this Packing was validated for another input length or device")
            pk = cu_seqlens
        else:
            cu = host_cu_seqlens(cu_seqlens, total, u.device)
            max_len = max(cu[i + 1] - cu[i] for i in range(len(cu) - 1))
            pk = Packing(cu, None, None, max_len, u.device)
        if pk.max_len > self.l_max:
            raise HyenaB200Error(f"a packed sequence of {pk.max_len} positions exceeds l_max = {self.l_max}{hint}")
        if max_seqlen is not None and int(max_seqlen) < pk.max_len:
            raise HyenaB200Error(f"max_seqlen = {int(max_seqlen)} is shorter than the longest sequence ({pk.max_len})")
        return pk

    def _packed_on_device(self, u, pk):
        if not u.is_cuda:
            raise HyenaB200Error("HyenaOperator (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        if pk.plan is None:
            pk.plan = ops.packed_plan(pk.cu)
            pk.tables = ops._bucket_tables(pk.plan, u.device)
        return pk

    def _forward_packed(self, u, pk, return_p=False):
        """forward(u, cu_seqlens=...): in_proj and out_proj as one B = 1 GEMM each over the packed tokens, the fused core
        per bucket of sequences (ops.PackedCoreFn: hyena_b200_core_fwd_packed / core_bwd_packed / short_bwd_packed).
        ``return_p``: -> (y, the in_proj output p (1, 3D, T) without its bias), for a packed prefill or admission."""
        if pk.total == 0 or pk.max_len == 0:
            return u * 0
        in_dtype, shape, total = u.dtype, u.shape, pk.total
        u32 = u.reshape(total, self.d_model).to(torch.float32)
        # the channel-major projection operands take their vector path at a length that is a multiple of 4: the packed
        # tensors get up to 3 trailing positions that belong to no sequence (zero in u, y_pre and dp)
        tp = -(-total // 4) * 4
        if tp != total:
            u32 = torch.nn.functional.pad(u32, (0, 0, 0, tp - total))
        k = self.filter_fn.filter_channel_major(pk.max_len)
        fb = self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias
        p = _InProj.apply(u32[None], self.in_proj.weight)                            # (1, 3D, tp)
        y_pre = ops.PackedCoreFn.apply(p, self.in_proj.bias, self.short_filter.weight, self.short_filter.bias, k, fb, pk)
        y = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias)[0, :total]
        y = y.reshape(shape).to(in_dtype)
        return (y, p) if return_p else y

    def check_packed_decode(self, u, cache, cu_seqlens, max_seqlen=None, lengths=None, rows=None):
        """Every host check of ``prefill(u, cache, cu_seqlens=..., max_seqlen=...)`` (``rows`` None) or of ``admit(u,
        cache, rows, cu_seqlens=...)`` without device work (Block and Backbone run it before their first kernel) -> (the
        operator's cache, Packing, the rows as a list)."""
        if lengths is not None:
            raise HyenaB200Error("cu_seqlens does not combine with lengths: packed prompts have no padding")
        what = "prefill" if rows is None else "admit"
        if not isinstance(cache, DecodeCache):
            raise HyenaB200Error(f"{what} needs a DecodeCache (allocate_decode_cache), got {type(cache).__name__}")
        c = cache.for_module(self)
        if u.requires_grad:
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        pk = self._packed_host(u, cu_seqlens, max_seqlen, self._prompt_hint(c, what))
        n = [pk.cu[i + 1] - pk.cu[i] for i in range(len(pk.cu) - 1)]
        if 0 in n:
            raise HyenaB200Error(f"{what}: packed prompt {n.index(0)} is empty; every prompt needs at least one position")
        P = pk.max_len
        if c.branched:
            raise HyenaB200Error(f"{what}: this cache is branched (DecodeCache.fork); packed prompts need a full cache")
        if rows is None:
            if c.t != 0:
                raise HyenaB200Error(f"prefill needs a fresh cache; this one is at position {c.t}")
            if len(n) != c.batch_size:
                raise HyenaB200Error(f"prefill: {len(n)} packed prompts for a decode cache of {c.batch_size} rows")
            if P > c.lcap:
                raise HyenaB200Error(f"prefill: a prompt of {P} positions exceeds Lcap = {c.lcap}")
        else:
            rows = _host_index(rows, c.batch_size, "admit: rows")
            if len(set(rows)) != len(rows):
                raise HyenaB200Error(f"admit: rows {rows} repeat a row")
            if len(rows) != len(n):
                raise HyenaB200Error(f"admit: {len(rows)} rows for {len(n)} packed prompts")
            ops.decode_admit_plan(c.t, c.lcap, P, c.win_b, c.win_wc)        # P <= Lcap, and the right shift fits
        pk = self._packed_on_device(u, pk)
        if not c.k.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; there is no CPU fallback")
        return c, pk, rows

    def check_lengths(self, u, lengths, cache=None, how="forward"):
        """Every host check of ``how``(u, [cache,] lengths=lengths) -- "forward", "prefill", "extend" or "step" -- without
        device work (Block and Backbone run it before their first kernel) -> the rows' first real positions."""
        if how == "step":
            self._no_ragged(lengths, "step")
        if how == "forward":
            if torch.is_grad_enabled() and (u.requires_grad or any(p.requires_grad for p in self.parameters())):
                raise HyenaB200Error("forward(u, lengths=...) is inference only (run under torch.no_grad()); to train on "
                                     "left-padded sequences pass their attention mask as forward(u, mask=...), or pad "
                                     "them on the right: the causal operator is exact there")
            starts = self._ragged_checks(u, lengths)
            if not u.is_cuda:
                raise HyenaB200Error("HyenaOperator (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
            return starts
        c = cache.for_module(self) if isinstance(cache, DecodeCache) else cache
        if how == "extend" and isinstance(c, DecodeCache) and (c.branched or c.t != 0):
            self._no_ragged(lengths, "extend on a cache that holds history or is branched")
        starts = self._ragged_checks(u, lengths, self._prompt_hint(c, "prefill") if isinstance(c, DecodeCache) else "")
        self._decode_checks(u, cache, u.shape[1], fresh=True)
        return starts

    def _forward_left_padded(self, u, lengths):
        starts = self.check_lengths(u, lengths)
        with torch.no_grad():
            row_start = torch.tensor(starts, dtype=torch.int32, device=u.device)
            y, _, _ = self._run_left_padded(u, row_start)
        return y

    def _run_left_padded(self, u, row_start):
        """Masked forward of a left-padded u (B, P, D) with row_start (B,) int32 on the device, under no_grad ->
        (y, p, g_o of the recurrences o >= 1 (order >= 3)).  Order 2: in_proj GEMM, the masked fused core
        (hyena_b200_core_fwd_rows), out_proj.  Order >= 3: the chained route with the pads zeroed in torch."""
        in_dtype, P = u.dtype, u.shape[1]
        u32 = u.to(torch.float32)
        k = self.filter_fn.filter_channel_major(P)
        fb = self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias
        if self.order == 2:
            p = _InProj.apply(u32, self.in_proj.weight).contiguous()
            C = self.short_filter.weight.shape[0]
            ib = self.in_proj.bias.contiguous() if self.in_proj.bias is not None else None
            y_pre, _, _ = ops.core_forward(p, ib, self.short_filter.weight.reshape(C, -1).contiguous(),
                                           self.short_filter.bias.contiguous(), ops.filter_spectrum(k),
                                           fb.reshape(-1).to(torch.float32).contiguous(), False, row_start)
            gs = []
        else:
            keep = torch.arange(P, device=u.device)[None, None, :] >= row_start.to(torch.long)[:, None, None]
            cap = {}
            y_pre = self._forward_chained(u32, k, fb, P, capture=cap, keep=keep)
            p, gs = cap["p"], cap["g"]
        y = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias).to(in_dtype)
        return y, p, gs

    def _forward_masked(self, u, pad):
        """forward(u, mask=...) under autograd: u (B, P, D) left-padded as ``pad`` (LeftPadding) says.  The in_proj input is
        zeroed at the pads (torch.where), so p is 0 there, du is 0 there and the pads stay out of d in_proj.weight whatever
        they hold.  Order 2 takes plain training's route choice with the masked core (hyena_b200_core_fwd_rows /
        core_bwd_rows); order >= 3 is the chained route with the pads masked, differentiable as it stands."""
        in_dtype, P = u.dtype, u.shape[1]
        row_start = pad.row_start
        keep = torch.arange(P, device=u.device)[None, :] >= row_start.to(torch.long)[:, None]          # (B, P)
        u32 = torch.where(keep[:, :, None], u.to(torch.float32), 0.0)
        k = self.filter_fn.filter_channel_major(P)
        fb = self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias
        if self.order > 2:
            y_pre = self._forward_chained(u32, k, fb, P, keep=keep[:, None, :])
        elif ops.proj_mode() == "tc":
            y_pre = ops.HyenaInCoreFn.apply(u32, self.in_proj.weight, self.in_proj.bias, self.short_filter.weight,
                                            self.short_filter.bias, k, fb, None, row_start)
        else:
            p = _InProj.apply(u32, self.in_proj.weight)
            y_pre = ops.HyenaCoreFn.apply(p, self.in_proj.bias, self.short_filter.weight, self.short_filter.bias, k, fb,
                                          None, row_start)
        return _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias).to(in_dtype)

    def _forward_chained(self, u, k, fb, l_filter, capture=None, keep=None):
        """order >= 3 (the shipped HyenaDNA layer default is 3, configs/model/layer/hyena_dna.yaml:3): the recurrence of
        hyena.py:414-423 as a chain of this library's long convolutions.  Projections and every FFT convolution
        (forward and backward) run on the sm_90a kernels; the gates and the 3-tap short filter between them are
        plain elementwise / depthwise torch ops here -- the fully fused pass exists for order 2 only.
        ``capture`` (a dict) receives the in_proj output "p" and the gated input "g" of every recurrence (prefill).
        ``keep`` ((B, 1, L) bool): left-padded rows; the short filter's input, every g and the output are zeroed where it is
        False (the masking of hyena_b200_core_fwd_rows)."""
        D, O1 = self.d_model, self.order - 1
        from .fftconv import fftconv_func
        p = _InProj.apply(u, self.in_proj.weight)                                   # (B, (order+1) D, l)
        if capture is not None:
            capture["p"], capture["g"] = p, []
        if l_filter < p.shape[-1]:
            p = p[..., :l_filter]
        p = p + self.in_proj.bias[None, :, None]
        if keep is not None:
            p = torch.where(keep, p, 0.0)
        uc = torch.nn.functional.conv1d(p, self.short_filter.weight, self.short_filter.bias,
                                        padding=self.short_filter_order - 1, groups=p.shape[1])[..., :l_filter]
        *x, v = uc.split(D, dim=1)
        kk = k.reshape(D, O1, l_filter)                                             # filter channels are ordered (v o): :408-412
        bb = fb.reshape(D, O1)
        bidir = self.filter_fn.bidirectional
        for o, x_i in enumerate(reversed(x[1:])):
            g = (v * x_i).contiguous()
            if keep is not None:
                g = torch.where(keep, g, 0.0).contiguous()
            if capture is not None:
                capture["g"].append(g)
            if bidir:
                from .fftconv import fftconv_ref
                v = fftconv_ref(g, kk[:, o].contiguous(), bb[:, o].contiguous(), None, gelu=False, bidirectional=True)
            else:
                v = fftconv_func(g, kk[:, o].contiguous(), bb[:, o].contiguous(), gelu=False)
        if keep is not None:
            return torch.where(keep, v * x[0], 0.0).contiguous()
        return (v * x[0]).contiguous()

    # ------------------------------------------------------------------------------ incremental decoding
    def allocate_decode_cache(self, batch_size, max_seqlen, history_dtype=torch.float32):
        """A DecodeCache for ``batch_size`` rows and up to min(max_seqlen, l_max) positions (decode.py), its history stored
        as ``history_dtype``: torch.float32, or torch.float16 / torch.bfloat16 for half the state (DESIGN.md section 4.16).
        ``max_seqlen`` None: an unbounded cache, which steps and extends past any position by sliding out the history the
        filter's l_max taps no longer reach (DESIGN.md section 4.20)."""
        return DecodeCache.allocate(self, batch_size, max_seqlen, history_dtype)

    @staticmethod
    def _prompt_hint(c, what):
        """The end of a too-long prompt's error for the cache ``c``: an unbounded cache points to extend."""
        return (f", the most an unbounded cache takes in one {what}; give it the first {c.reach} positions and extend by "
                "the rest") if c.unbounded else ""

    @classmethod
    def _check_prompt(cls, c, P, what):
        """An unbounded cache takes prompts of at most l_max positions (the filter's reach) in one prefill or admit."""
        if c.unbounded and P > c.reach:
            raise HyenaB200Error(f"{what}: a prompt of {P} positions exceeds l_max = {c.reach}{cls._prompt_hint(c, what)}")

    def _decode_checks(self, u, cache, n, fresh=False):
        if not isinstance(cache, DecodeCache):
            raise HyenaB200Error(f"decoding needs a DecodeCache (allocate_decode_cache), got {type(cache).__name__}")
        c = cache.for_module(self)
        if u.requires_grad:
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        if self.filter_fn.bidirectional:
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        if u.dim() != 3 or u.shape[-1] != self.d_model or u.shape[1] != n:
            raise HyenaB200Error(f"decoding input must be (B, {n}, {self.d_model}); got {tuple(u.shape)}")
        if u.shape[0] != c.batch_size:
            raise HyenaB200Error(f"batch size {u.shape[0]} differs from the decode cache's {c.batch_size}")
        if fresh and c.branched:
            raise HyenaB200Error("prefill needs a fresh cache; this one is branched (DecodeCache.fork)")
        if fresh and c.t != 0:
            raise HyenaB200Error(f"prefill needs a fresh cache; this one is at position {c.t}")
        if c.branched and c.t + n > c.base + c.hc:
            raise HyenaB200Error(f"decoding past the branch horizon: positions [{c.t}, {c.t + n}) exceed base + Hc = "
                                 f"{c.base} + {c.hc} = {c.base + c.hc} (fork with a larger horizon, up to Lcap = {c.lcap})")
        if c.unbounded:
            if fresh:
                self._check_prompt(c, n, "prefill")
        elif c.t + n > c.lcap:
            raise HyenaB200Error(f"decoding past the cache: positions [{c.t}, {c.t + n}) exceed Lcap = min(max_seqlen, "
                                 f"l_max) = {c.lcap} (l_max = {self.l_max}: the filter has no taps beyond it)")
        if not u.is_cuda or not c.k.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; there is no CPU fallback")
        return c

    def _decode_params(self):
        C = self.short_filter.weight.shape[0]
        return (self.in_proj.bias.detach().contiguous() if self.in_proj.bias is not None else None,
                self.short_filter.weight.detach().reshape(C, -1).contiguous(), self.short_filter.bias.detach().contiguous())

    def prefill(self, u, cache, lengths=None, cu_seqlens=None, max_seqlen=None):
        """Run the first P positions, u (B, P, D), and fill ``cache`` (which must be fresh) for stepping.  The output is
        the one ``forward(u)`` gives, bit for bit: the same kernels run in the same order.

        ``lengths`` (B integers in [1, P]): prompts of different lengths, left-padded to P; row b's real tokens are its
        positions [P - lengths[b], P).  Pad positions enter neither the outputs nor the cache: the output at a real position
        and everything decoded after the prefill are those of the unpadded row; the output at a pad position is
        out_proj(0) = out_proj.bias.  Every row ends at position P, so the rows step together; row b can hold at most
        Lcap - (P - lengths[b]) real positions.  ``forward(u, lengths=...)`` gives the same outputs, bit for bit.

        ``cu_seqlens`` ((N+1,) integer cumulative lengths, as for ``forward``; N = the cache's batch size): u (total, D) or
        (1, total, D) holds N prompts of at least one position packed back to back, prompt i going into row i.  The output
        has u's shape and the bits of ``forward(u, cu_seqlens=...)``; the cache is left bit for bit as ``prefill`` of the
        same prompts left-padded to the longest, P, with ``lengths`` leaves it: every row ends at position P (DESIGN.md
        section 4.19).  ``max_seqlen``, when given, must be at least P."""
        if cu_seqlens is not None:
            return self._prefill_packed(u, cache, cu_seqlens, max_seqlen, lengths)
        if lengths is not None:
            return self._prefill_left_padded(u, cache, lengths)
        c = self._decode_checks(u, cache, u.shape[1] if u.dim() == 3 else -1, fresh=True)
        with torch.no_grad():
            P = u.shape[1]
            y, p, gs = self._prefill_run(u)
            ib, sw, sb = self._decode_params()
            ops.decode_hist(p.contiguous(), ib, sw, sb, c)
            for o in range(1, self.order - 1):
                c.h[o, :, :, :P].copy_(gs[o])
            c.t = P
            c.reset_window()
        return y

    def _prefill_run(self, u):
        """The forward of an unpadded u (B, P, D) as prefill runs it, under no_grad -> (y, the in_proj output p without its
        bias, g_o of the recurrences o >= 1 (order >= 3))."""
        in_dtype = u.dtype
        u32 = u.to(torch.float32)
        P = u32.shape[1]
        if self.order == 2:
            y = self.forward(u)
            y = y[0] if isinstance(y, tuple) else y
            # the in_proj output the forward consumed (the projections are deterministic: same bits)
            if ops.proj_mode() == "tc":
                p = ops.proj_gemm(u32.contiguous(), 0, self.in_proj.weight.contiguous(), False, 0)
            else:
                p = _InProj.apply(u32, self.in_proj.weight)
            gs = []
        else:                               # forward's order >= 3 route, keeping its intermediates
            k = self.filter_fn.filter_channel_major(P)
            fb = self.filter_fn.bias if self.filter_fn.use_bias else 0 * self.filter_fn.bias
            cap = {}
            y_pre = self._forward_chained(u32, k, fb, P, capture=cap)
            y = _OutProj.apply(y_pre, self.out_proj.weight, self.out_proj.bias).to(in_dtype)
            p, gs = cap["p"], cap["g"]
        return y, p, gs

    def check_admit(self, u, cache, rows, lengths=None):
        """Every host check of ``admit(u, cache, rows, lengths)`` without device work (Block and Backbone run it before
        their first kernel) -> (the operator's cache, the rows as a list, the prompts' first real positions)."""
        if not isinstance(cache, DecodeCache):
            raise HyenaB200Error(f"admit needs a DecodeCache (allocate_decode_cache), got {type(cache).__name__}")
        c = cache.for_module(self)
        if c.branched:
            raise HyenaB200Error("admit: this cache is branched; admission, release and compaction need a full cache")
        if u.requires_grad:
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        if self.filter_fn.bidirectional:
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        if u.dim() != 3 or u.shape[-1] != self.d_model or u.shape[0] < 1 or u.shape[1] < 1:
            raise HyenaB200Error(f"admit: prompts must be (k, P, {self.d_model}); got {tuple(u.shape)}")
        k, P = u.shape[0], u.shape[1]
        rows = _host_index(rows, c.batch_size, "admit: rows")
        if len(set(rows)) != len(rows):
            raise HyenaB200Error(f"admit: rows {rows} repeat a row")
        if len(rows) != k:
            raise HyenaB200Error(f"admit: {len(rows)} rows for {k} prompts")
        starts = [P - n for n in host_lengths(lengths, k, P)] if lengths is not None else [0] * k
        self._check_prompt(c, P, "admit")
        ops.decode_admit_plan(c.t, c.lcap, P, c.win_b, c.win_wc)        # P <= Lcap, and the right shift fits
        if not u.is_cuda or not c.k.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; there is no CPU fallback")
        return c, rows, starts

    def admit(self, u, cache, rows, lengths=None, cu_seqlens=None):
        """Prompts join a running cache: u (k, P, D) goes into the cache rows ``rows`` (k distinct rows, typically ones
        freed by ``DecodeCache.release``) -> y (k, P, D), the bits ``prefill`` of u gives on a fresh k-row cache.  Each
        prompt is placed so that it ends at the cache's position t, with a zero history before it, so its row decodes
        exactly as after that prefill while the other rows go on unchanged (DESIGN.md section 4.15).  When P > t the whole
        cache first shifts right by P - t rounded up to a multiple of 4 (at t = 0 the position becomes P, and every row
        that takes no prompt is free).  ``lengths`` (k integers in [1, P]): the prompts are left-padded, as for prefill.
        The other rows' history, tail and window are not touched; an open window stays open (the admitted rows' part of
        it is recomputed).  Every row can hold up to Lcap - (t - m) more positions after a ``compact`` by m: the room is
        bounded by the longest live row, not by the row's own length.

        ``cu_seqlens``: the k prompts packed back to back, as for ``prefill``; P is the longest.  The output has u's shape
        and the bits of ``forward(u, cu_seqlens=...)``; each admitted row is left bit for bit as ``admit`` of the prompts
        left-padded to P leaves it."""
        if cu_seqlens is not None:
            return self._admit_packed(u, cache, rows, cu_seqlens, lengths)
        c, rows, starts = self.check_admit(u, cache, rows, lengths)
        P = u.shape[1]
        with torch.no_grad():
            if lengths is None:
                row_start = None
                y, p, gs = self._prefill_run(u)
            else:
                row_start = torch.tensor(starts, dtype=torch.int32, device=u.device)
                y, p, gs = self._run_left_padded(u, row_start)
            c._admit_clock(P)
            ib, sw, sb = self._decode_params()
            ops.decode_admit(p.contiguous(), ib, sw, sb, gs, c, rows, row_start)
            c._took(rows, [c.t - P + s for s in starts])
        return y

    def _prefill_packed(self, u, cache, cu_seqlens, max_seqlen, lengths):
        c, pk, _ = self.check_packed_decode(u, cache, cu_seqlens, max_seqlen, lengths)
        with torch.no_grad():
            y, p = self._forward_packed(u, pk, return_p=True)
            P, cu = pk.max_len, pk.cu
            c.t = P
            c.set_start([P - (cu[i + 1] - cu[i]) for i in range(len(cu) - 1)])
            ib, sw, sb = self._decode_params()
            seg_base = torch.tensor([x - P for x in cu[1:]], dtype=torch.int64, device=u.device)
            ops.decode_admit_packed(p, ib, sw, sb, c, list(range(len(cu) - 1)), seg_base, c.start_dev, P)
            c.reset_window()
        return y

    def _admit_packed(self, u, cache, rows, cu_seqlens, lengths):
        c, pk, rows = self.check_packed_decode(u, cache, cu_seqlens, None, lengths, rows)
        with torch.no_grad():
            y, p = self._forward_packed(u, pk, return_p=True)
            P, cu = pk.max_len, pk.cu
            n = [cu[i + 1] - cu[i] for i in range(len(cu) - 1)]
            c._admit_clock(P)
            ib, sw, sb = self._decode_params()
            seg_base = torch.tensor([x - P for x in cu[1:]], dtype=torch.int64, device=u.device)
            row_start = torch.tensor([P - m for m in n], dtype=torch.int32, device=u.device)
            ops.decode_admit_packed(p, ib, sw, sb, c, rows, seg_base, row_start, P)
            c._took(rows, [c.t - m for m in n])
        return y

    def _prefill_left_padded(self, u, cache, lengths):
        starts = self.check_lengths(u, lengths, cache, "prefill")
        c = cache.for_module(self)
        with torch.no_grad():
            c.set_start(starts)
            y, p, gs = self._run_left_padded(u, c.start_dev)
            ib, sw, sb = self._decode_params()
            ops.decode_hist(p.contiguous(), ib, sw, sb, c, row_start=c.start_dev)
            P = u.shape[1]
            for o in range(1, self.order - 1):
                c.h[o, :, :, :P].copy_(gs[o])
            c.t = P
            c.reset_window()
        return y

    @staticmethod
    def _no_ragged(lengths, what):
        if lengths is not None:
            raise HyenaB200Error(f"{what} takes no lengths: left-padded prompts are prefilled together on a fresh cache, and "
                                 "rows then advance together (ragged appends would need per-row positions)")

    def step(self, u_t, cache, lengths=None):
        """One position: u_t (B, 1, D) -> y (B, 1, D), the output at position ``cache.t``; advances the cache.  Stepping a
        fresh cache starts the sequence (empty history).  The in_proj / out_proj products of one position are fp32
        matrix-vector products (F.linear); the operator itself runs in csrc/decode.cuh, two launches per recurrence.  After
        a run of steps at a long history the step reads only the positions of a window opened by one FFT refresh
        (ops.decode_window_plan chooses).  On a branched cache (DecodeCache.fork) the step reads each branch's positions since
        the fork base only (ops.decode_branch_step).  An unbounded cache at Lcap slides first (DecodeCache._make_room)."""
        self._no_ragged(lengths, "step")
        c = self._decode_checks(u_t, cache, 1)
        c._make_room(1, step=True)
        y = self._step_with(u_t, c, ops.decode_branch_step if c.branched else ops.decode_step_auto)
        c.t += 1
        return y

    def _step_with(self, u_t, c, core):
        """The work of step on the operator's cache ``c`` with ``core`` (one of the ops.decode_*step functions) for the
        operator itself; no checks and no position advance (StepGraph captures this with the device-position steps)."""
        with torch.no_grad():
            in_dtype = u_t.dtype
            B, D = u_t.shape[0], self.d_model
            u = u_t.to(torch.float32).reshape(B, D)
            p_t = torch.nn.functional.linear(u, self.in_proj.weight).contiguous()          # bias added in the kernel
            ib, sw, sb = self._decode_params()
            y_pre = core(p_t, ib, sw, sb, c)
            y = torch.nn.functional.linear(y_pre, self.out_proj.weight, self.out_proj.bias)
        return y.reshape(B, 1, D).to(in_dtype)

    def capture_step(self, cache, batch_size=None, dtype=torch.float32):
        """A decode.StepGraph: ``step`` on ``cache`` captured in CUDA graphs and replayed one position at a time."""
        return StepGraph(self, cache, batch_size, dtype)

    def extend(self, u, cache, lengths=None):
        """n >= 1 more positions at once: u (B, n, D) -> y (B, n, D), the outputs at positions [cache.t, cache.t + n);
        advances the cache by n.  On a fresh cache this is ``prefill`` (bit-identical to ``forward``).  Otherwise in_proj and
        out_proj of the chunk run on the wgmma projection GEMM and every recurrence on csrc/decode_extend.cuh: the direct
        Toeplitz kernel over the cached history, or for large n the FFT convolution of the whole history
        (ops.decode_extend_uses_fft chooses from t and n).  On a branched cache the same routes run over each branch's
        positions since the fork base only (ops.decode_branch_extend).  ``lengths`` is accepted on a fresh cache only,
        where this is ``prefill(u, cache, lengths)``.  An unbounded cache slides first when the n positions would pass
        Lcap, and runs more than S positions (l_max on a fresh cache) as consecutive extends (DESIGN.md section 4.20)."""
        n = u.shape[1] if u.dim() == 3 else -1
        if n < 1:
            raise HyenaB200Error(f"extend input must be (B, n, {self.d_model}) with n >= 1; got {tuple(u.shape)}")
        if lengths is not None:
            self.check_lengths(u, lengths, cache, "extend")
            return self.prefill(u, cache, lengths)
        c = self._decode_checks(u, cache, n)
        if c.branched:
            return self._extend(u, c, ops.decode_branch_extend)
        if c.unbounded and n > (c.slide if c.t else c.reach):
            return self._extend_pieces(u, c)
        if c.t == 0:
            return self.prefill(u, c)
        c._make_room(n)
        return self._extend(u, c, ops.decode_extend)

    def _extend_pieces(self, u, c):
        """extend of the unbounded operator cache ``c`` by more positions than it takes at once: consecutive extends of at
        most S positions (the first a prefill of at most l_max on a fresh cache), each after its own slide, written into
        one output tensor."""
        B, n, D = u.shape
        y, i = None, 0
        while i < n:
            m = min(n - i, c.slide if c.t else c.reach)
            yi = self.extend(u[:, i:i + m].contiguous(), c)
            if y is None:
                y = torch.empty(B, n, D, dtype=yi.dtype, device=yi.device)
            y[:, i:i + m] = yi
            i += m
        return y

    def _extend(self, u, c, core):
        """extend on a non-fresh cache with ``core`` (ops.decode_extend or one of its two routes) for the operator."""
        with torch.no_grad():
            in_dtype, n = u.dtype, u.shape[1]
            p = ops.proj_gemm(u.to(torch.float32).contiguous(), 0, self.in_proj.weight.detach().contiguous(), False, 0)
            ib, sw, sb = self._decode_params()
            y_pre = core(p, ib, sw, sb, c)                                              # (B, D, n)
            b = self.out_proj.bias.detach().contiguous() if self.out_proj.bias is not None else None
            y = ops.proj_gemm(y_pre, 1, self.out_proj.weight.detach().contiguous(), False, 1, bias=b)
            c.t += n
            c.steps = 0
        return y.to(in_dtype)

    @property
    def d_output(self):
        return self.d_model
