"""Windowed decoding steps: the C ABI and its guards, the route rule (ops.decode_window_plan / decode_step_auto with the
device work stubbed) and the window identity in fp64, following the cache layout the kernels use (no GPU needed)."""
import ctypes
from importlib import import_module

import numpy as np
import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")

P = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def test_win_step_abi_present():
    L = _lib.lib()
    name = "hyena_b200_decode_win_step"
    assert name in _lib.SIGNATURES and hasattr(L, name)
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        assert name + "(" in f.read()
    assert L.hyena_b200_abi_version() == 2
    names = [L.hyena_b200_kind_name(i).decode() for i in range(L.hyena_b200_kind_count())]
    assert names[-1] == "decode_win_step" and names.count("decode_win_step") == 1
    assert names[-4:-1] == ["decode_extend_hist", "decode_extend_dot", "decode_extend_combine"]


def _win(p_t=P, h=P, k=P, win=P, v_in=None, o=0, order=2, t=20, b=16, Wc=8, W=8, Lcap=64, B=1, cache_B=1):
    return _lib.lib().hyena_b200_decode_win_step(p_t, P, P, P, k, P, h, P, P, v_in, P, P, win, B, cache_B, 8, order, o, t,
                                                 b, Wc, W, Lcap, None)


def test_win_step_abi_guards():
    assert _win(win=None) != 0 and "null pointer" in _err()
    assert _win(p_t=None) != 0 and "recurrence 0 needs" in _err()
    assert _win(o=1, order=3) != 0 and "v_in" in _err()
    assert _win(o=1) != 0 and "recurrence" in _err()
    assert _win(b=18, t=20) != 0 and "multiple of 4" in _err()
    assert _win(b=-4) != 0 and "multiple of 4" in _err()
    assert _win(t=15) != 0 and "outside the window" in _err()                 # t < b
    assert _win(t=24) != 0 and "outside the window" in _err()                 # t = b + Wc
    assert _win(Wc=0) != 0 and "outside the decode cache" in _err()
    assert _win(Wc=9, W=8) != 0 and "outside the decode cache" in _err()
    assert _win(b=60, t=60, Wc=8, W=8) != 0 and "outside the decode cache" in _err()   # b + Wc > Lcap
    assert _win(B=2) != 0 and "differs from the decode cache" in _err()
    assert _win(Lcap=(1 << 20) + 1) != 0 and "exceeds the supported maximum" in _err()
    assert _win(h=ctypes.c_void_p(260)) != 0 and "aligned" in _err()


def _ops():
    import hyena_dna_b200 as H
    return H.ops


def test_plan_thresholds():
    ops = _ops()
    T, S = ops.WINDOW_MIN_T, ops.WINDOW_AFTER_STEPS
    lcap = 1 << 20
    assert ops.decode_window_plan(T, lcap, S) == "refresh"
    assert ops.decode_window_plan(T - 1, lcap, S) == "plain"
    assert ops.decode_window_plan(T, lcap, S - 1) == "plain"
    assert ops.decode_window_plan(lcap - 1, lcap, 10 ** 6) == "refresh"
    assert ops.decode_window_plan(0, lcap, 0) == "plain"


def test_plan_window_and_expiry():
    ops = _ops()
    T, S, W = ops.WINDOW_MIN_T, ops.WINDOW_AFTER_STEPS, ops.WINDOW
    lcap = 1 << 20
    b, wc = ops.decode_window_bounds(T + 6, lcap)
    assert (b, wc) == (T + 4, W)
    for t in (b, b + 1, b + wc - 1):
        assert ops.decode_window_plan(t, lcap, S, b, wc) == "window"
        assert ops.decode_window_plan(t, lcap, 0, b, wc) == "window"          # an extend inside the window keeps it
    assert ops.decode_window_plan(b + wc, lcap, S + wc, b, wc) == "refresh"    # expired while stepping: refresh at once
    assert ops.decode_window_plan(b + wc, lcap, 0, b, wc) == "plain"          # expired after an extend: count again
    assert ops.decode_window_plan(b - 1, lcap, S, b, wc) == "refresh"         # before the window (rewound cache)


def test_window_bounds_alignment_and_clipping():
    ops = _ops()
    W = ops.WINDOW
    for t in range(100, 108):
        b, wc = ops.decode_window_bounds(t, 1 << 20)
        assert b % 4 == 0 and b <= t < b + 4 and wc == W
    lcap = 5003
    for t in (lcap - W - 3, lcap - 10, lcap - 1):
        b, wc = ops.decode_window_bounds(t, lcap)
        assert b % 4 == 0 and b <= t < b + wc and b + wc == min(b + W, lcap)
    assert ops.decode_window_bounds(lcap - 1, lcap) == (lcap - 3, 3)


def _cpu_cache(op, B=1, lcap=None):
    import hyena_dna_b200 as H
    lcap = lcap or op.l_max
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    return H.DecodeCache(op, B, lcap, lcap, torch.zeros(F * ld + 4), torch.zeros(F), torch.zeros(O - 1, B, D, ld),
                         torch.zeros(B, C, 2), torch.zeros(B, C), torch.zeros(B, D, (lcap + 1023) // 1024))


def _stub_routes(monkeypatch, ops, log):
    def refresh(c):
        c.win_b, c.win_wc = ops.decode_window_bounds(c.t, c.lcap)
        log.append("refresh")
    monkeypatch.setattr(ops, "decode_window_refresh", refresh)
    monkeypatch.setattr(ops, "decode_step", lambda *a: log.append("plain"))
    monkeypatch.setattr(ops, "decode_win_step", lambda *a: log.append("window"))


def test_step_auto_counts_and_resets(monkeypatch):
    """Steps count up; a window opens after WINDOW_AFTER_STEPS of them; an extend resets the count but keeps a valid
    window; a prefill resets both (device work stubbed)."""
    import hyena_dna_b200 as H
    ops = H.ops
    monkeypatch.setattr(ops, "WINDOW_MIN_T", 8)
    monkeypatch.setattr(ops, "WINDOW_AFTER_STEPS", 3)
    monkeypatch.setattr(ops, "WINDOW", 8)
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op)
    log = []
    _stub_routes(monkeypatch, ops, log)

    def steps(n):
        for _ in range(n):
            ops.decode_step_auto(None, None, None, None, c)
            c.t += 1

    c.t = 5
    steps(6)                                     # t = 5..7 below WINDOW_MIN_T; at t = 8 the count is 3: refresh
    assert log == ["plain"] * 3 + ["refresh"] + ["window"] * 3 and (c.win_b, c.win_wc) == (8, 8) and c.steps == 6
    # an extend of 2 (device work stubbed): the count restarts, the window [8, 16) stays valid
    monkeypatch.setattr(ops, "proj_gemm", lambda act, al, W, wt, ol, bias=None, **kw: torch.zeros(
        (act.shape[0], W.shape[0], act.shape[1]) if ol == 0 else (act.shape[0], act.shape[2], W.shape[0])))
    op._extend(torch.zeros(1, 2, 8), c, lambda p, ib, sw, sb, cc: torch.zeros(1, 8, 2))
    assert c.t == 13 and c.steps == 0 and (c.win_b, c.win_wc) == (8, 8)
    log.clear()
    steps(5)                                     # t = 13..15 in the window; at 16 it has expired and the count is 3
    assert log == ["window"] * 3 + ["refresh", "window", "window"]
    assert (c.win_b, c.win_wc) == (16, 8)
    # a prefill starts a new sequence: window closed, count 0
    monkeypatch.setattr(op, "_decode_checks", lambda u, cache, n, fresh=False: cache)
    monkeypatch.setattr(op, "forward", lambda u: torch.zeros(1, u.shape[1], 8))
    monkeypatch.setattr(ops, "decode_hist", lambda *a: None)
    c.t = 0
    op.prefill(torch.zeros(1, 4, 8), c)
    assert c.t == 4 and c.steps == 0 and c.win_wc == 0
    assert c.window_nbytes == 0


def test_window_nbytes_of_a_stack():
    import hyena_dna_b200 as H
    op = H.HyenaOperator(8, 64, emb_dim=5, order=3)
    a, b = _cpu_cache(op, B=2), _cpu_cache(op, B=2)
    s = H.DecodeCache.stack([a, b])
    assert s.window_nbytes == 0
    a.win_f = torch.zeros(2, 2, 8, 16)
    assert a.window_nbytes == s.window_nbytes == 4 * 2 * 2 * 8 * 16
    assert a.nbytes == H.DecodeCache.layout_nbytes(2, 8, 3, 64)            # the window is not part of the layout


# ---------------------------------------------------------------------------------------------- window identity (fp64)
def _layout(k, lcap):
    """k (D, lcap) -> the cache's reversed rows (D, ld) (k[j] at ld-1-j)."""
    D = k.shape[0]
    ld = (lcap + 3) // 4 * 4
    krev = torch.zeros(D, ld, dtype=k.dtype)
    krev[:, ld - lcap:] = k.flip(-1)
    return krev, ld


def _refresh(krev, ld, h, b, wc):
    """F (B, D, wc) as ops._history_conv builds it: un-reversed taps [0, b + wc), history [0, b) zero-padded, causal FFT
    convolution (here numpy fp64), outputs [b, b + wc)."""
    L = b + wc
    k = krev[:, ld - L:].flip(-1).numpy()
    u = np.zeros(h.shape[:2] + (L,))
    u[:, :, :b] = h[:, :, :b].numpy()
    n = 2 * L
    conv = np.fft.irfft(np.fft.rfft(u, n) * np.fft.rfft(k, n)[None], n)[..., :L]
    return torch.from_numpy(conv[:, :, b:].copy())


def _win_out(krev, ld, h, bias, F, b, t):
    """out[t] the way the windowed step computes it: decode_dot_kernel on h + b with t - b (k[t-s] = krev[ld-1-(t-b)+(s-b)]),
    F[t-b], then (k[0] + bias) g[t]."""
    j = t - b
    hw = h[:, :, b:]
    dot = (hw[:, :, :j] * krev[None, :, ld - 1 - j:ld - 1]).sum(-1)
    return dot + F[:, :, j] + (krev[None, :, ld - 1] + bias[None]) * h[:, :, t]


def _direct(k, h, bias, t):
    return (h[:, :, :t + 1] * k[None, :, :t + 1].flip(-1)).sum(-1) + bias[None] * h[:, :, t]


@pytest.mark.parametrize("lcap,b,W", [(300, 0, 64), (300, 4, 64), (3000, 1500, 512), (5001, 2052, 1024),
                                      (3001, 2900, 512)])
def test_window_identity_fp64(lcap, b, W):
    """For t = b, b + 1, b + Wc - 1 and a few inside: the windowed sum equals the direct O(t) sum.  Covers b = 0, b not a
    multiple of 1024 and a window clipped at Lcap (the last case: Wc = 101)."""
    g = torch.Generator().manual_seed(lcap + b)
    B, D = 2, 3
    k = torch.randn(D, lcap, generator=g, dtype=torch.float64) / (1 + torch.arange(lcap, dtype=torch.float64)) ** 0.5
    h = torch.randn(B, D, lcap, generator=g, dtype=torch.float64)
    bias = torch.randn(D, generator=g, dtype=torch.float64)
    wc = min(W, lcap - b)
    krev, ld = _layout(k, lcap)
    hl = torch.zeros(B, D, ld, dtype=torch.float64)
    hl[:, :, :lcap] = h
    poisoned = hl.clone()
    poisoned[:, :, b:] = 1e3                     # positions >= b must not reach F
    F = _refresh(krev, ld, poisoned, b, wc)
    for t in sorted({b, b + 1, b + wc // 2, b + wc - 2, b + wc - 1}):
        want = _direct(k, h, bias, t)
        got = _win_out(krev, ld, hl, bias, F, b, t)
        torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)
