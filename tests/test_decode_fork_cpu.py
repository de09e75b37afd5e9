"""Branched decode caches (DecodeCache.fork / select): the C ABI and its guards, host validation and bookkeeping with the
device work stubbed, the branch identity in fp64 and a model of the shifted-pointer index arithmetic of the reused dot
kernels (no GPU needed)."""
import ctypes
from importlib import import_module

import numpy as np
import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")

P = ctypes.c_void_p(256)          # never dereferenced: the checks come first
NAMES = ["hyena_b200_decode_branch_step", "hyena_b200_decode_branch_extend_hist", "hyena_b200_decode_branch_extend_dot",
         "hyena_b200_decode_branch_combine"]


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def test_branch_abi_present():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header
    assert L.hyena_b200_abi_version() == 3
    names = [L.hyena_b200_kind_name(i).decode() for i in range(L.hyena_b200_kind_count())]
    assert names[-1] == "decode_win_step" and len(names) == 33          # branch launches count under existing kinds


def _step(p_t=P, h=P, k=P, f=P, parent=P, v_in=None, o=0, order=2, t=21, b=16, Hc=8, H=8, Lcap=64, R=1):
    return _lib.lib().hyena_b200_decode_branch_step(p_t, P, P, P, k, P, h, P, P, v_in, P, P, f, parent, R, 8, order, o, t,
                                                    b, Hc, H, Lcap, None)


def _hist(p=P, h=P, t=16, n=4, b=16, Hc=8, H=8, Lcap=64):
    return _lib.lib().hyena_b200_decode_branch_extend_hist(p, P, P, P, h, P, P, 1, 8, 2, t, n, b, Hc, H, Lcap, None)


def _dot(h=P, k=P, groups=None, t=17, n=4, b=16, Hc=8, H=8, Lcap=64):
    if groups is None:
        groups = _lib.lib().hyena_b200_decode_extend_groups(1, 8, t - b, n)
    return _lib.lib().hyena_b200_decode_branch_extend_dot(h, k, P, groups, 1, 8, 2, 0, t, n, b, Hc, H, Lcap, None)


def _comb(f=P, parent=P, groups=1, t=17, n=4, b=16, Hc=8, H=8, Lcap=64, o=0):
    return _lib.lib().hyena_b200_decode_branch_combine(P, 4, 1, groups, P, P, P, P, f, parent, 1, 8, 2, o, t, n, b, Hc, H,
                                                       Lcap, None)


def test_branch_step_guards():
    assert _step(f=None) != 0 and "null pointer" in _err()
    assert _step(parent=None) != 0 and "null pointer" in _err()
    assert _step(p_t=None) != 0 and "recurrence 0 needs" in _err()
    assert _step(o=1, order=3) != 0 and "v_in" in _err()
    assert _step(o=1) != 0 and "recurrence" in _err()
    assert _step(b=18, t=20) != 0 and "multiple of 4" in _err()
    assert _step(b=-4) != 0 and "multiple of 4" in _err()
    assert _step(Hc=0) != 0 and "outside the decode cache" in _err()
    assert _step(b=60, t=60, Hc=8, H=8) != 0 and "outside the decode cache" in _err()      # b + Hc > Lcap
    assert _step(H=6) != 0 and "history width" in _err()                                     # not a multiple of 4
    assert _step(Hc=8, H=4, t=17) != 0 and "history width" in _err()                         # H < Hc
    assert _step(b=16, Hc=40, H=52, t=17) != 0 and "history width" in _err()                 # H > ld - b: k would underflow
    assert _step(t=15) != 0 and "outside the branch horizon" in _err()                       # t < b
    assert _step(t=24) != 0 and "outside the branch horizon" in _err()                       # t = b + Hc
    assert _step(R=0) != 0 and "bad shape" in _err()
    assert _step(Lcap=(1 << 20) + 1) != 0 and "exceeds the supported maximum" in _err()
    assert _step(h=ctypes.c_void_p(260)) != 0 and "aligned" in _err()
    assert _step(k=ctypes.c_void_p(260)) != 0 and "aligned" in _err()


def test_branch_extend_guards():
    assert _hist(p=None) != 0 and "null pointer" in _err()
    assert _hist(n=0) != 0 and "outside the branch horizon" in _err()
    assert _hist(t=20, n=5) != 0 and "outside the branch horizon" in _err()                 # t + n = b + Hc + 1
    assert _hist(t=20, n=4, Hc=8, H=4) != 0 and "history width" in _err()
    assert _dot(groups=7) != 0 and "partials sized" in _err()
    assert _dot(k=ctypes.c_void_p(264)) != 0 and "aligned" in _err()
    assert _dot(b=12, t=17) != 0 and "outside the branch horizon" in _err()                 # t + n past b + Hc
    assert _comb(f=None) != 0 and "null pointer" in _err()
    assert _comb(parent=None) != 0 and "null pointer" in _err()
    assert _comb(groups=0) != 0 and "bad partial layout" in _err()
    assert _comb(o=1) != 0 and "recurrence" in _err()
    assert _comb(Lcap=20, b=16, Hc=8) != 0 and "outside the decode cache" in _err()


# ---------------------------------------------------------------------------------------------- host side (device stubbed)
def _H():
    import hyena_dna_b200 as H
    return H


def _cpu_cache(op, B=2, lcap=64, t=0, seed=0):
    H = _H()
    g = torch.Generator().manual_seed(seed)
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    c = H.DecodeCache(op, B, lcap, lcap, torch.randn(F * ld + 4, generator=g), torch.randn(F, generator=g),
                      torch.randn(O - 1, B, D, ld, generator=g), torch.randn(B, C, 2, generator=g), torch.zeros(B, C),
                      torch.zeros(B, D, (lcap + 1023) // 1024))
    c.t = t
    return c


def _conv_stub(calls):
    """ops._history_conv in fp64 on the CPU (direct sums), logging its calls."""
    def conv(cache, ld, h, o, hist, L):
        calls.append((o, hist, L, h.shape[0]))
        D, O = cache.d_model, cache.order
        k = cache.k[:(O - 1) * D * ld].view(D, O - 1, ld)[:, o, ld - L:].flip(-1).double()
        u = torch.zeros(h.shape[0], D, L, dtype=torch.float64)
        u[:, :, :hist] = h[:, :, :hist].double()
        out = torch.zeros_like(u)
        for t in range(L):
            out[:, :, t] = (u[:, :, :t + 1] * k[None, :, :t + 1].flip(-1)).sum(-1)
        return out.float()
    return conv


@pytest.fixture
def stubbed(monkeypatch):
    H = _H()
    calls = []
    monkeypatch.setattr(H.ops, "_history_conv", _conv_stub(calls))
    return calls


@pytest.mark.parametrize("t0,lcap,horizon", [(1, 64, 16), (3, 64, 16), (4, 64, 16), (17, 64, 16), (18, 64, 16),
                                             (19, 64, 16), (23, 64, 5), (50, 61, 4096), (60, 61, 16)])
def test_fork_bookkeeping(stubbed, t0, lcap, horizon):
    """(b, Hc, H) for every t0 mod 4, t0 < 4 (b = 0: no F computed) and a horizon clipped at Lcap; the copied history and
    tails, the parent index, F of each distinct parent row, shared filter, nbytes."""
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5, order=3)
    c = _cpu_cache(op, B=3, lcap=lcap, t=t0)
    rows = [2, 0, 2, 2]
    br = c.fork(rows, horizon)
    b, hc, W = H.ops.decode_branch_bounds(t0, lcap, horizon)
    assert b == t0 - t0 % 4 and W % 4 == 0 and W >= hc
    assert hc == min((horizon + 3) // 4 * 4, lcap - b) and hc > t0 - b
    assert br.branched and not c.branched and (br.base, br.hc, br.t, br.batch_size) == (b, hc, t0, 4)
    assert br.k is c.k and br.bias is c.bias
    assert tuple(br.h.shape) == (2, 4, 8, W) and tuple(br.f.shape) == (2, 2, 8, W)
    assert tuple(br.part.shape) == (4, 8, (W + 1023) // 1024)
    assert br.parent.dtype == torch.int32 and br.parent.tolist() == [1, 0, 1, 1]
    for i, r in enumerate(rows):
        assert torch.equal(br.h[:, i, :, :t0 - b], c.h[:, r, :, b:t0])
        assert torch.equal(br.tail[i], c.tail[r])
    assert not br.h[:, :, :, t0 - b:].any()
    if b == 0:
        assert stubbed == [] and not br.f.any()
    else:
        assert stubbed == [(0, b, b + hc, 2), (1, b, b + hc, 2)]
        for o in range(2):
            for p, r in enumerate([0, 2]):
                want = _conv_stub([])(c, c.h.shape[-1], c.h[o, [r]], o, b, b + hc)[0, :, b:]
                assert torch.equal(br.f[o, p, :, :hc], want)
    own = (br.h, br.f, br.tail, br.s_t, br.part, br.parent)
    assert br.nbytes == sum(x.numel() * x.element_size() for x in own)
    assert c.nbytes == H.DecodeCache.layout_nbytes(3, 8, 3, lcap)
    # a snapshot: the parent's history and tail can change without touching the branches
    before = br.h.clone(), br.tail.clone()
    c.h.add_(1.0)
    c.tail.add_(1.0)
    assert torch.equal(br.h, before[0]) and torch.equal(br.tail, before[1])


def test_fork_validates_on_the_host(stubbed, monkeypatch):
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op, B=2, t=9)
    monkeypatch.setattr(H.ops, "decode_fork", lambda *a: pytest.fail("device work before validation"))
    for rows, msg in [([], "empty"), ([2], r"outside \[0, 2\)"), ([0, -1], r"outside \[0, 2\)"), ([0.5], "integers"),
                      (torch.zeros(1, 1, dtype=torch.long), "1-D"), (torch.tensor([1.0]), "1-D"), ([True], "integers"),
                      ("01", "integers")]:
        with pytest.raises(H.HyenaB200Error, match=msg):
            c.fork(rows)
    with pytest.raises(H.HyenaB200Error, match="horizon"):
        c.fork([0], 0)
    c.t = 0
    with pytest.raises(H.HyenaB200Error, match="1 <= t0"):
        c.fork([0])
    c.t = 64
    with pytest.raises(H.HyenaB200Error, match="1 <= t0"):
        c.fork([0])
    c.t = 9
    monkeypatch.setattr(op.filter_fn, "bidirectional", True)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        c.fork([0])


def test_select_and_stack(stubbed):
    H = _H()
    ops_a, ops_b = H.HyenaOperator(8, 64, emb_dim=5), H.HyenaOperator(8, 64, emb_dim=5)
    s = H.DecodeCache.stack([_cpu_cache(ops_a, B=2, t=22, seed=1), _cpu_cache(ops_b, B=2, t=22, seed=2)])
    br = s.fork([1, 0, 1], horizon=12)
    assert br.branched and br.t == 22 and len(br.layers) == 2
    la = br.for_module(ops_a)
    assert la.owner is ops_a and la.batch_size == 3 and (la.base, la.hc) == (20, 12)
    with pytest.raises(H.HyenaB200Error, match="branched already"):
        br.fork([0])
    with pytest.raises(H.HyenaB200Error, match="not branched"):
        s.select([0])
    for idx, msg in [([], "empty"), ([3], "outside"), ([[0]], "integers")]:
        with pytest.raises(H.HyenaB200Error, match=msg):
            br.select(idx)
    la.h[:, :, :, 2:5] = torch.arange(3.0)[None, :, None, None]          # distinct suffix rows per branch
    la.t = 25
    sel = br.select(torch.tensor([2, 2, 0, 1]))
    ls = sel.for_module(ops_a)
    assert ls.batch_size == 4 and ls.t == 25 and ls.f is la.f and ls.k is la.k
    assert ls.parent.tolist() == [la.parent[i].item() for i in (2, 2, 0, 1)]
    for i, r in enumerate((2, 2, 0, 1)):
        assert torch.equal(ls.h[:, i], la.h[:, r]) and torch.equal(ls.tail[i], la.tail[r])
    assert sel.nbytes == sum(c.nbytes for c in sel.layers)


def test_horizon_and_prefill_checks(stubbed):
    """One position past base + Hc raises before any device work and names the horizon; prefill on a branch raises."""
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op, B=1, t=10)
    br = c.fork([0, 0], horizon=8)                          # b = 8, Hc = 8: positions [8, 16)
    assert (br.base, br.hc) == (8, 8)
    u = torch.zeros(2, 1, 8)
    br.t = 16
    h0 = br.h.clone()
    for call in (lambda: op.step(u, br), lambda: op.extend(torch.zeros(2, 2, 8), br), lambda: op(u, inference_params=br)):
        with pytest.raises(H.HyenaB200Error, match="horizon"):
            call()
    assert br.t == 16 and torch.equal(br.h, h0)
    br.t = 14
    with pytest.raises(H.HyenaB200Error, match="horizon"):
        op.extend(torch.zeros(2, 3, 8), br)
    with pytest.raises(H.HyenaB200Error, match="branched"):
        op.prefill(torch.zeros(2, 3, 8), br)
    with pytest.raises(H.HyenaB200Error, match="batch size"):
        op.step(torch.zeros(1, 1, 8), br)


# ---------------------------------------------------------------------------------------------- the identity (fp64)
def _recurrence(k, bias, v, xs):
    """Direct causal recurrence in fp64: k (O-1, D, L), bias (O-1, D), v (B, D, L), xs (O-1+1 gates) -> y (B, D, L) and
    the gated inputs g_o (B, D, L) of every recurrence."""
    O1 = k.shape[0]
    L = v.shape[-1]
    g, gs = v * xs[O1], []
    for o in range(O1):
        gs.append(g)
        out = np.zeros_like(g)
        for t in range(L):
            out[:, :, t] = (g[:, :, :t + 1] * k[o][None, :, t::-1]).sum(-1) + bias[o][None] * g[:, :, t]
        g = out * xs[O1 - 1 - o]
    return g, gs


@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("t0,lcap,horizon", [(2, 80, 16), (40, 80, 16), (41, 80, 16), (42, 80, 9), (43, 80, 16),
                                             (77, 79, 64)])
def test_branch_identity_fp64(order, t0, lcap, horizon):
    """F (from the parent's history before b) + the branch's own sum over [b, t) + (k[0] + bias) g[t] equals the full causal
    recurrence of prefix || branch suffix at every branch position, for every recurrence of order 2 and 3."""
    ops = _H().ops
    rng = np.random.default_rng(t0 * 7 + order)
    D, O1 = 3, order - 1
    b, hc, _ = ops.decode_branch_bounds(t0, lcap, horizon)
    L = b + hc
    k = rng.standard_normal((O1, D, lcap)) / np.sqrt(1 + np.arange(lcap))
    bias = rng.standard_normal((O1, D))
    par_v, par_x = rng.standard_normal((1, D, L)), rng.standard_normal((order, 1, D, L))
    br_v, br_x = rng.standard_normal((2, D, L)), rng.standard_normal((order, 2, D, L))
    br_v[:, :, :t0], br_x[:, :, :, :t0] = par_v[:, :, :t0], par_x[:, :, :, :t0]    # both branches continue the parent
    _, pg = _recurrence(k, bias, par_v, list(par_x))
    want, _ = _recurrence(k, bias, br_v, list(br_x))
    # the branched computation: F from the parent's g_o[0, b), the branch rows from b on
    n2 = 2 * L
    F = [np.fft.irfft(np.fft.rfft(np.where(np.arange(L) < b, pg[o], 0), n2) * np.fft.rfft(k[o][:, :L], n2)[None], n2)
         [..., b:L] for o in range(O1)]
    h = [np.zeros((2, D, hc)) for _ in range(O1)]
    for o in range(O1):
        h[o][:, :, :t0 - b] = pg[o][:, :, b:t0]
    got = np.zeros((2, D, L))
    for t in range(t0, L):
        j = t - b
        g = br_v[:, :, t] * br_x[O1][:, :, t]
        for o in range(O1):
            h[o][:, :, j] = g
            out = F[o][:, :, j] + (h[o][:, :, :j] * k[o][None, :, j:0:-1]).sum(-1) + (k[o][:, 0] + bias[o])[None] * g
            g = out * br_x[O1 - 1 - o][:, :, t]
        got[:, :, t] = g
    np.testing.assert_allclose(got[:, :, t0:], want[:, :, t0:L], rtol=1e-9, atol=1e-9)


# ---------------------------------------------------------------------------------------------- shifted-pointer model
def _dot_model(ld, H, t, b):
    """decode_dot_kernel on a branch row: h' = branch row (stride H), t' = t - b, filter pointer k + ld - H.  Returns the
    absolute filter indices of the loads and, per used (masked-in) history position s = b + s', the tap index."""
    tp = t - b
    R = (H - 1 - tp) & 3
    kb = (ld - H) + (H - 1 - tp - R)                 # absolute offset of kb in the row
    loads, used = [], {}
    for s0 in range(0, tp, 4):                       # the s0 < t test; chunks and lanes enumerate every multiple of 4
        ka = kb + s0 + np.arange(4)
        loads += list(ka) + (list(ka + 4) if R else [])
        for i in range(4):
            if s0 + i < tp:                          # hv masked at positions >= t'
                used[b + s0 + i] = kb + s0 + R + i
    return loads, used


@pytest.mark.parametrize("ld,t,b,H", [(64, 21, 16, 8), (64, 23, 20, 44), (1028, 1027, 1024, 4), (4096, 3000, 1100, 2996),
                                      (4096, 4093, 0, 4096), (2052, 2050, 4, 2048), (2052, 2049, 1024, 1028)])
def test_dot_kernel_shifted_indices(ld, t, b, H):
    loads, used = _dot_model(ld, H, t, b)
    assert sorted(used) == list(range(b, t))
    for s, idx in used.items():
        assert idx == ld - 1 - t + s                # k[t-s] at the same absolute element as the unbranched call
    assert all(0 <= i < ld + 4 for i in loads)      # within the row or the next row / the 4 floats of padding
    assert (ld - H) % 4 == 0 and ((ld - H) + (H - 1 - (t - b) - ((H - 1 - (t - b)) & 3))) % 4 == 0


def _ext_dot_model(ld, H, t, n, b, NT):
    """decode_ext_dot_kernel on a branch row: window A4 = H - t' - j0 + s0 - NT - R of the shifted row, staged as zero
    where idx < 0 or idx >= H; output j = j0 + r at position s' = s0 + q reads window index q + NT - 1 - r + R.  Checks every
    (j, s') pair the kernel multiplies with a non-zero history value."""
    tp = t - b
    Lp, R = tp + n, (-tp) & 3
    for j0 in range(0, n, NT):
        for s0 in range(0, Lp, 1024):
            if s0 > tp + j0 + NT - 1:
                break
            A4 = H - tp - j0 + s0 - NT - R
            assert A4 % 4 == 0
            r = np.arange(NT)[:, None]
            q = np.arange(1024)[None, :]
            wi = q + NT - 1 - r + R
            assert wi.min() >= 0 and wi.max() < 1024 + NT + 4
            idx = A4 + wi
            j, sp = j0 + r + 0 * q, s0 + q + 0 * r
            live = sp < Lp                           # staged history is zero from t' + n on
            m = t + j - (b + sp)                     # the tap the pair needs
            staged = (idx >= 0) & (idx < H)
            absolute = (ld - H) + idx
            ok = live & (j < n)
            assert np.all(staged[ok & (m >= 0)]) and np.all(absolute[ok & (m >= 0)] == (ld - 1 - m)[ok & (m >= 0)])
            assert not np.any(staged[ok & (m < 0)])  # the idx < H test is the causal mask
            assert np.all(j[live & (idx < 0)] >= n)  # the idx >= 0 test zeroes taps of outputs past n only


@pytest.mark.parametrize("ld,t,n,b,H", [(64, 21, 3, 16, 8), (64, 17, 27, 16, 44), (2052, 1030, 1, 1028, 1024),
                                        (2052, 1031, 9, 1028, 1024), (4096, 2999, 65, 1100, 2996),
                                        (4096, 3003, 600, 1100, 2996), (4096, 5, 4091, 4, 4092), (2048, 1, 64, 0, 2048)])
def test_ext_dot_kernel_shifted_indices(ld, t, n, b, H):
    assert t + n <= b + H <= ld
    for NT in (8, 64):
        _ext_dot_model(ld, H, t, n, b, NT)
