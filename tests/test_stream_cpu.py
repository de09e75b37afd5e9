"""Streaming forward (``forward(u, stream=True)``; DESIGN.md section 4.21) without a GPU: the window and chunk plan, the
guards of the two window entry points, the host validation of HyenaOperator, Block and Backbone, each firing before any
device work, and a self-check that the streaming truth the GPU tests use rejects a plan with too little context."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

_lib = import_module("hyena_dna_b200._lib")
ops = import_module("hyena_dna_b200.ops")

PTR = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


# ---------------------------------------------------------------------------------------------- helpers of the GPU tests
def causal_conv(g, k, bias, n_fft=None):
    """c[..., t] = sum_{j < Lk} k[c, j] g[..., t - j] + bias[c] g[..., t] over the whole of g (B, C, L), by FFT in g's
    dtype (torch.fft on g's device), a channel block at a time."""
    B, C, L = g.shape
    Lk = k.shape[-1]
    n = n_fft or 1 << (L + Lk - 1).bit_length()
    out = torch.empty_like(g)
    step = max(1, (1 << 24) // (B * n))
    for c0 in range(0, C, step):
        c1 = min(C, c0 + step)
        kf = torch.fft.rfft(k[c0:c1].to(g.dtype), n=n)
        out[:, c0:c1] = torch.fft.irfft(torch.fft.rfft(g[:, c0:c1], n=n) * kf, n=n)[..., :L]
    return out + bias.to(g.dtype)[None, :, None] * g


def stream_truth(op, u, dtype=torch.float64, positions=None):
    """The operator's composition with its l_max-tap causal convolution over the whole sequence (what an unbounded
    DecodeCache gives), in ``dtype`` on u's device: u (B, L, D) -> y (B, L, D).  ``positions``: return y at these
    positions only (the output projection runs on them alone)."""
    D, O1, Lk = op.d_model, op.order - 1, op.l_max
    with torch.no_grad():
        k = op.filter_fn.filter_channel_major(Lk).detach().to(u.device, dtype)
        fb = (op.filter_fn.bias if op.filter_fn.use_bias else 0 * op.filter_fn.bias).detach().to(u.device, dtype)
        Win, bin_ = op.in_proj.weight.to(u.device, dtype), op.in_proj.bias.to(u.device, dtype)
        p = torch.einsum("bld,cd->bcl", u.to(dtype), Win) + bin_[None, :, None]
        L = p.shape[-1]
        uc = F.conv1d(p, op.short_filter.weight.to(u.device, dtype), op.short_filter.bias.to(u.device, dtype),
                      padding=2, groups=p.shape[1])[..., :L]
        del p
        *x, v = uc.split(D, dim=1)
        kk, bb = k.reshape(D, O1, Lk), fb.reshape(D, O1)
        for o, x_i in enumerate(reversed(x[1:])):
            v = causal_conv(v * x_i, kk[:, o], bb[:, o])
        yp = v * x[0]
        if positions is not None:
            yp = yp[..., positions]
        y = torch.einsum("bcl,dc->bld", yp, op.out_proj.weight.to(u.device, dtype)) + op.out_proj.bias.to(u.device, dtype)
    return y


def windowed_core(p, k, bias, sw, sb, wins, L_b):
    """A model of hyena_b200_core_fwd_windows on one channel (fp64, torch): y_pre of the gated core for p (3, n) (x0, x1,
    v rows with their in_proj bias) on the windows ``wins`` (stream_windows of a row of n positions), each window alone:
    positions before row_start read zeros, and only positions from out_start are stored."""
    n = p.shape[-1]
    y = torch.full((n,), float("nan"), dtype=p.dtype)
    for start, rs, os_ in wins:
        t = torch.arange(L_b) + start
        pw = torch.where((torch.arange(L_b) >= rs)[None, :], p[:, t.clamp(0, n - 1)], 0.0)
        s = F.conv1d(pw[None], sw[:, None, :], sb, padding=2, groups=3)[0, :, :L_b]
        c = causal_conv((s[1] * s[2])[None, None], k[None], bias[None])[0, 0]
        y[t[os_:]] = (c * s[0])[os_:]
    return y


def direct_core(p, k, bias, sw, sb):
    """The same y_pre over the whole row at once (fp64)."""
    n = p.shape[-1]
    s = F.conv1d(p[None], sw[:, None, :], sb, padding=2, groups=3)[0, :, :n]
    return causal_conv((s[1] * s[2])[None, None], k[None], bias[None])[0, 0] * s[0]


# ---------------------------------------------------------------------------------------------- the plan
def _check_row(wins, n, L_b, c):
    """Every position of a row of n stored by exactly one window, each later window with >= c positions of context."""
    hits = torch.zeros(n, dtype=torch.int64)
    for i, (start, rs, os_) in enumerate(wins):
        assert 0 <= rs <= os_ < L_b
        assert rs == max(0, -start)
        lo, hi = start + os_, start + L_b
        assert 0 <= lo < hi <= n
        hits[lo:hi] += 1
        if i == 0:
            assert start <= 0 and os_ == rs               # the row's first window starts it, without context
        else:
            assert start >= 0 and os_ >= c
    assert bool((hits == 1).all())


def _check_plan(pl, L):
    assert ops.STREAM_MIN_WINDOW <= pl.L_b <= ops.STREAM_MAX_WINDOW and pl.L_b & (pl.L_b - 1) == 0
    assert pl.L_b > pl.context
    hits = torch.zeros(L, dtype=torch.int64)
    for s, a, e in pl.chunks:
        assert 0 <= s <= a < e <= L
        assert s == 0 or a - s >= pl.chunk_context
        hits[a:e] += 1
        _check_row(pl.windows(e - s), e - s, pl.L_b, pl.context)
    assert bool((hits == 1).all())


@pytest.mark.parametrize("L,l_max,order,B", [
    (1026 + 1, 1026, 2, 1), (3 * 1026 + 5, 1026, 2, 3), ((1 << 20) + 1, 1026, 2, 3), ((1 << 21) + 3, 1026, 3, 3),
    ((1 << 20) + 1, 4099, 2, 1), ((1 << 21) + 3, 1 << 16, 2, 3), ((1 << 21) + 3, 1 << 16, 3, 3),
    (3 * 61 + 5, 61, 3, 3), ((1 << 23) + 5, 1026, 2, 1), (3 * 1000002, 1000002, 2, 1), ((1 << 20) + 7, (1 << 20) - 2, 2, 1),
])
def test_plan_table(L, l_max, order, B):
    pl = ops.stream_plan(L, l_max, order, B)
    _check_plan(pl, L)
    assert pl.context == (l_max + 1 if order == 2 else l_max - 1)
    assert pl.chunk_context == ops.stream_context(l_max, order)
    if order >= 3:
        assert pl.chunk_context == (order - 1) * (l_max - 1) + 2


def test_plan_exhaustive_small():
    for l_max in (1, 2, 3, 7, 61, 500, 1021, 1022):
        for order in (2, 3, 4):
            c = ops.stream_context(l_max, 2 if order == 2 else 1)
            for L in list(range(1, 40)) + [1023, 1024, 1025, 2047, 2048, 2049, 3 * 1024 + 1, 5000]:
                for cp in (None, 1, 3000):
                    if c >= 1024:
                        continue
                    _check_plan(ops.stream_plan(L, l_max, order, 1, L_b=1024, chunk_positions=cp), L)


def test_plan_window_length_rule_and_errors():
    assert ops.stream_window_length(62) == 1 << 16
    assert ops.stream_window_length(1027) == 1 << 16
    assert ops.stream_window_length(32771) == 1 << 18
    assert ops.stream_window_length((1 << 16) + 1) == 1 << 19
    assert ops.stream_window_length(1000003) == 1 << 20
    for L, l_max, order, B, L_b in [((1 << 20) - 5, 1026, 2, 3, 1 << 20), (1 << 20, 32770, 3, 3, 1 << 20),
                                    (1027, 1026, 2, 1, 2048), (63, 61, 2, 2, 1024), (5000, 4099, 3, 1, 8192)]:
        pl = ops.stream_plan(L, l_max, order, B)                        # fits: one chunk of one window
        assert pl.L_b == L_b and pl.chunks == [(0, 0, L)] and len(pl.windows(L)) == 1
    pl = ops.stream_plan((1 << 20) + 1, 1026, 2, 3)
    assert pl.L_b == 1 << 16 and len(pl.chunks) > 1
    with pytest.raises(_lib.HyenaB200Error, match="leaves no room"):
        ops.stream_plan(10, (1 << 20) - 1, 2)
    with pytest.raises(_lib.HyenaB200Error, match="power of two"):
        ops.stream_plan(5000, 61, 2, L_b=1536)
    with pytest.raises(_lib.HyenaB200Error, match="power of two"):
        ops.stream_plan(5000, 2000, 2, L_b=1024)
    with pytest.raises(_lib.HyenaB200Error, match="bad shape"):
        ops.stream_plan(0, 61, 2)


def test_window_launches_split_at_65535():
    for rows in (1, 65535, 65536, 3 * 65535 + 2):
        parts = list(ops._window_launches(rows))
        assert all(0 < n <= 65535 for _, n in parts)
        assert [r0 for r0, _ in parts] == list(range(0, rows, 65535)) and sum(n for _, n in parts) == rows


def test_tables_address_rows_back_to_back():
    wins = ops.stream_windows(5000, 1024, 62)
    sb, rs, os_ = ops.stream_tables(wins, 3, 7000, torch.device("cpu"))
    assert sb.dtype == torch.int64 and rs.dtype == torch.int32 and os_.dtype == torch.int32
    assert sb.tolist() == [b * 7000 + w[0] for b in range(3) for w in wins]
    assert os_.tolist() == [w[2] for w in wins] * 3


# ---------------------------------------------------------------------------------------------- C guards
def test_window_entry_point_guards():
    L = _lib.lib()
    core = lambda sb, rs, os_, total, B, D, Lb: L.hyena_b200_core_fwd_windows(
        PTR, None, PTR, PTR, PTR, PTR, PTR, sb, rs, os_, total, B, D, Lb, PTR, 1 << 30, None)
    conv = lambda sb, rs, os_, total, B, D, Lb: L.hyena_b200_fftconv_fwd_windows(
        PTR, PTR, PTR, PTR, sb, rs, os_, total, B, D, Lb, PTR, 1 << 30, None)
    n0 = _lib.launch_count()
    for fn in (core, conv):
        assert fn(PTR, PTR, PTR, 1 << 20, 1, 8, (1 << 20) + 1) != 0 and "exceeds the supported maximum" in _err()
        assert fn(PTR, PTR, PTR, 1 << 20, 65536, 8, 1024) != 0 and "too large" in _err()
        assert fn(PTR, PTR, PTR, 0, 1, 8, 1024) != 0 and "bad packed length" in _err()
        assert fn(PTR, PTR, None, 1 << 20, 1, 8, 1024) != 0 and "out_start" in _err()
        assert fn(PTR, PTR, ctypes.c_void_p(258), 1 << 20, 1, 8, 1024) != 0 and "out_start" in _err()
        assert fn(None, PTR, PTR, 1 << 20, 1, 8, 1024) != 0 and "null pointer" in _err()
        assert fn(ctypes.c_void_p(260), PTR, PTR, 1 << 20, 1, 8, 1024) != 0 and "seg_base" in _err()
    rc = L.hyena_b200_core_fwd_windows(PTR, None, PTR, PTR, PTR, PTR, None, PTR, PTR, PTR, 1 << 20, 1, 8, 1024, PTR,
                                       1 << 30, None)
    assert rc != 0 and "null pointer" in _err()
    rc = L.hyena_b200_fftconv_fwd_windows(PTR, ctypes.c_void_p(260), PTR, PTR, PTR, PTR, PTR, 1 << 20, 1, 8, 1024, PTR,
                                          1 << 30, None)
    assert rc != 0 and "kspec" in _err()
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- host validation
def _op(**kw):
    H = _H()
    return H.HyenaOperator(8, kw.pop("l_max", 64), emb_dim=5, **kw)


def test_operator_validation_before_device_work():
    H = _H()
    op = _op()
    u = torch.zeros(2, 200, 8)
    n0 = _lib.launch_count()
    with pytest.raises(H.HyenaB200Error, match="inference only"):
        op(u, stream=True)
    with torch.no_grad():
        for kw, msg in [(dict(lengths=[4, 6]), "lengths, mask or cu_seqlens"),
                        (dict(mask=torch.ones(2, 200)), "lengths, mask or cu_seqlens"),
                        (dict(cu_seqlens=torch.tensor([0, 200])), "lengths, mask or cu_seqlens"),
                        (dict(inference_params=H.DecodeCache()), "DecodeCache")]:
            with pytest.raises(H.HyenaB200Error, match=msg):
                op(u, stream=True, **kw)
        with pytest.raises(H.HyenaB200Error, match="bidirectional"):
            _op(bidirectional=True)(u, stream=True)
        for bad in (torch.zeros(200, 8), torch.zeros(2, 200, 7), torch.zeros(2, 0, 8)):
            with pytest.raises(H.HyenaB200Error, match="stream=True takes u"):
                op(bad, stream=True)
        big = H.HyenaOperator(2, (1 << 20) - 1, emb_dim=5)
        with pytest.raises(H.HyenaB200Error, match="leaves no room"):
            big(torch.zeros(1, 4, 2), stream=True)
        for o in (2, 3):
            with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):      # every check passes: the device is next
                _op(order=o)(u, stream=True)
            with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
                _op(order=o)(u[:, :10], stream=True)
    x = torch.zeros(1, 200, 8, requires_grad=True)
    with pytest.raises(H.HyenaB200Error, match="inference only"):
        op(x, stream=True)
    assert _lib.launch_count() == n0


def test_block_and_backbone_validate_before_device_work():
    H = _H()
    from hyena_dna_b200.mlp import Mlp
    mixer = partial(H.HyenaOperator, l_max=64, emb_dim=5)
    blk = H.Block(8, mixer_cls=mixer)
    bb = H.Backbone(8, 2, mixer, mlp_cls=partial(Mlp, hidden_features=32))
    u = torch.zeros(2, 300, 8)
    n0 = _lib.launch_count()
    with pytest.raises(H.HyenaB200Error, match="inference only"):
        blk(u, mixer_kwargs={"stream": True})
    with pytest.raises(H.HyenaB200Error, match="inference only"):
        bb(u, stream=True)
    with torch.no_grad():
        with pytest.raises(H.HyenaB200Error, match="lengths, mask or cu_seqlens"):
            blk(u, mixer_kwargs={"stream": True}, lengths=[3, 4])
        with pytest.raises(H.HyenaB200Error, match="lengths, mask or cu_seqlens"):
            bb(u, stream=True, mask=torch.ones(2, 300))
        bb.layers[1].mixer.filter_fn.bidirectional = True            # a later layer's error fires before layer 0 runs
        with pytest.raises(H.HyenaB200Error, match="bidirectional"):
            bb(u, stream=True)
        bb.layers[1].mixer.filter_fn.bidirectional = False
        with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
            bb(u, stream=True)
        with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
            blk(u, mixer_kwargs={"stream": True})
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- truth self-check
@pytest.mark.parametrize("l_max", [5, 61])
def test_truth_rejects_a_plan_with_one_position_too_little_context(l_max):
    g = torch.Generator().manual_seed(l_max)
    n, L_b = 3500, 1024
    p = torch.randn(3, n, generator=g, dtype=torch.float64)
    k = torch.randn(l_max, generator=g, dtype=torch.float64)
    bias = torch.randn(1, generator=g, dtype=torch.float64)[0]
    sw = torch.randn(3, 3, generator=g, dtype=torch.float64)
    sb = torch.randn(3, generator=g, dtype=torch.float64)
    truth = direct_core(p, k, bias, sw, sb)
    c = ops.stream_context(l_max, 2)
    good = windowed_core(p, k, bias, sw, sb, ops.stream_windows(n, L_b, c), L_b)
    assert torch.isfinite(good).all()
    assert float((good - truth).abs().max()) <= 1e-9 * float(truth.abs().max())
    bad = windowed_core(p, k, bias, sw, sb, ops.stream_windows(n, L_b, c - 1), L_b)
    assert float((bad - truth).abs().max()) > 1e-3 * float(truth.abs().max())


def test_stream_truth_is_the_operator_below_l_max():
    """Up to l_max the streaming truth is the plain operator (its fp64 oracle composition): a check of stream_truth."""
    H = _H()
    torch.manual_seed(0)
    op = H.HyenaOperator(4, 64, emb_dim=5)
    u = torch.randn(2, 50, 4, dtype=torch.float64)
    k = torch.randn(4, 64)
    op.filter_fn.filter_channel_major = lambda L: k[:, :L]
    y = stream_truth(op, u)
    # the reference recurrence: fftconv over L positions with the first L taps
    p = u @ op.in_proj.weight.double().T + op.in_proj.bias.double()
    s = F.conv1d(p.transpose(1, 2), op.short_filter.weight.double(), op.short_filter.bias.double(), padding=2,
                 groups=12)[..., :50]
    x0, x1, v = s.split(4, dim=1)
    g = x1 * v
    c = torch.zeros_like(g)
    for t in range(50):
        for j in range(t + 1):
            c[..., t] += k[:, j].double() * g[..., t - j]
    c = c + op.filter_fn.bias.double()[None, :, None] * g
    ref = (c * x0).transpose(1, 2) @ op.out_proj.weight.double().T + op.out_proj.bias.double()
    assert float((y - ref).abs().max()) < 1e-10
