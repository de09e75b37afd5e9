"""Extending a decode cache by n positions: the C ABI, the guards of the Python API, the dispatch of
forward(..., inference_params=cache) and the direct/FFT selection rule (no GPU needed: every call below is rejected before
any CUDA work, or runs with the decoding entry points stubbed)."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


P = ctypes.c_void_p(256)          # never dereferenced: the checks come first
NAMES = ("hyena_b200_decode_extend_groups", "hyena_b200_decode_extend_hist", "hyena_b200_decode_extend_dot",
         "hyena_b200_decode_extend_combine")


def test_extend_abi_present():
    L = _lib.lib()
    for name in NAMES:
        assert name in _lib.SIGNATURES and hasattr(L, name)
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert name + "(" in header
    assert L.hyena_b200_abi_version() == 2
    names = [L.hyena_b200_kind_name(i).decode() for i in range(L.hyena_b200_kind_count())]
    assert {"decode_extend_hist", "decode_extend_dot", "decode_extend_combine"} <= set(names)


def test_extend_groups():
    L = _lib.lib()
    assert L.hyena_b200_decode_extend_groups(0, 8, 0, 1) == 0 and L.hyena_b200_decode_extend_groups(1, 8, 0, 0) == 0
    for B, D, t, n in [(1, 256, 1 << 14, 1), (1, 256, (1 << 20) - 64, 64), (9, 32, 100, 3), (2, 64, 3001, 511)]:
        g = L.hyena_b200_decode_extend_groups(B, D, t, n)
        nchunk = -(-(t + n) // 1024)
        assert 1 <= g <= nchunk
        cpb = -(-nchunk // g)
        assert -(-nchunk // cpb) == g                      # every group holds at least one chunk


def _hist(p=P, h=P, tail=P, s=P, B=1, cache_B=1, order=2, t=0, n=4, Lcap=64):
    return _lib.lib().hyena_b200_decode_extend_hist(p, P, P, P, h, tail, s, B, cache_B, 8, order, t, n, Lcap, None)


def _dot(h=P, k=P, part=P, groups=None, B=1, cache_B=1, o=0, order=2, t=10, n=4, Lcap=64):
    g = _lib.lib().hyena_b200_decode_extend_groups(B, 8, t, n) if groups is None else groups
    return _lib.lib().hyena_b200_decode_extend_dot(h, k, part, g, B, cache_B, 8, order, o, t, n, Lcap, None)


def _comb(part=P, groups=1, out=P, o=0, order=2, t=10, n=4, Lcap=64, B=1, cache_B=1):
    return _lib.lib().hyena_b200_decode_extend_combine(part, 4, 1, groups, P, P, P, out, B, cache_B, 8, order, o, t, n, Lcap,
                                                       None)


def test_extend_abi_guards():
    assert _hist(p=None) != 0 and "null pointer" in _err()
    assert _hist(s=None) != 0 and "null pointer" in _err()
    assert _hist(t=60, n=5) != 0 and "outside the decode cache" in _err()
    assert _hist(n=0) != 0 and "n must be >= 1" in _err()
    assert _hist(B=2) != 0 and "differs from the decode cache" in _err()
    assert _hist(order=1) != 0 and "order" in _err()
    assert _dot(k=None) != 0 and "null pointer" in _err()
    assert _dot(groups=1000) != 0 and "groups" in _err()
    assert _dot(o=1) != 0 and "recurrence" in _err()
    assert _dot(t=61, n=4) != 0 and "outside the decode cache" in _err()
    assert _dot(h=ctypes.c_void_p(260)) != 0 and "aligned" in _err()
    assert _comb(out=None) != 0 and "null pointer" in _err()
    assert _comb(groups=0) != 0 and "groups" in _err()
    assert _comb(o=2, order=3) != 0 and "recurrence" in _err()
    assert _comb(Lcap=(1 << 20) + 1) != 0 and "exceeds the supported maximum" in _err()


def _op(**kw):
    import hyena_dna_b200 as H
    return H.HyenaOperator(8, 64, emb_dim=5, **kw)


def _cpu_cache(op, B=2, lcap=None):
    """A cache with the layout's shapes on the CPU (allocate_decode_cache itself needs the GPU)."""
    import hyena_dna_b200 as H
    lcap = lcap or op.l_max
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    return H.DecodeCache(op, B, lcap, lcap, torch.zeros(F * ld + 4), torch.zeros(F), torch.zeros(O - 1, B, D, ld),
                         torch.zeros(B, C, 2), torch.zeros(B, C), torch.zeros(B, D, (lcap + 1023) // 1024))


def test_extend_guards():
    import hyena_dna_b200 as H
    op = _op()
    c = _cpu_cache(op)
    c.t = 10
    u = torch.zeros(2, 5, 8)
    with pytest.raises(H.HyenaB200Error, match="requires grad"):
        op.extend(u.clone().requires_grad_(True), c)
    with pytest.raises(H.HyenaB200Error, match="CUDA"):              # everything else is valid: the CPU tensor is the fault
        op.extend(u, c)
    with pytest.raises(H.HyenaB200Error, match="batch size 3"):
        op.extend(torch.zeros(3, 5, 8), c)
    with pytest.raises(H.HyenaB200Error, match=r"\(B, n, 8\) with n >= 1"):
        op.extend(torch.zeros(2, 0, 8), c)
    with pytest.raises(H.HyenaB200Error, match=r"\(B, n, 8\) with n >= 1"):
        op.extend(torch.zeros(5, 8), c)
    with pytest.raises(H.HyenaB200Error, match=r"\(B, 5, 8\)"):
        op.extend(torch.zeros(2, 5, 7), c)
    with pytest.raises(H.HyenaB200Error, match="DecodeCache"):
        op.extend(u, {"not": "a cache"})
    with pytest.raises(H.HyenaB200Error, match="not allocated for this"):
        _op().extend(u, c)
    c.t = 60                                                           # Lcap = l_max = 64: 4 positions left
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        op.extend(u, c)
    assert c.t == 60
    opb = _op(bidirectional=True)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        opb.extend(u, _cpu_cache(opb))


def test_block_and_backbone_extend_guards():
    import hyena_dna_b200 as H
    m = H.Backbone(8, 2, partial(H.HyenaOperator, l_max=64, emb_dim=5))
    with pytest.raises(H.HyenaB200Error, match="requires grad"):
        m.extend(torch.zeros(1, 4, 8, requires_grad=True), None)
    with pytest.raises(H.HyenaB200Error, match="requires grad"):
        m.layers[0].extend(torch.zeros(1, 4, 8, requires_grad=True), None, None)


@pytest.mark.parametrize("t,n,want", [(0, 1, "step"), (0, 2, "prefill"), (0, 100, "prefill"), (5, 1, "step"),
                                      (5, 2, "extend"), (63, 1, "step"), (1, 63, "extend")])
def test_forward_dispatch(t, n, want):
    """forward(u, inference_params=cache): fresh cache and n > 1 -> prefill, n == 1 -> step, otherwise extend (the three
    entry points stubbed on the instance)."""
    op = _op()
    c = _cpu_cache(op)
    c.t = t
    calls = []
    for name in ("prefill", "step", "extend"):
        setattr(op, name, lambda u, cache, name=name: calls.append((name, cache)) or u)
    y = op(torch.zeros(2, n, 8), inference_params=c)
    assert calls == [(want, c)] and y.shape == (2, n, 8)


def test_forward_dispatch_reaches_extend_checks():
    """Unstubbed: several positions on a non-fresh cache reach extend, whose CPU-tensor check is the error."""
    import hyena_dna_b200 as H
    op = _op()
    c = _cpu_cache(op)
    c.t = 7
    with pytest.raises(H.HyenaB200Error, match="CUDA"):
        op(torch.zeros(2, 3, 8), inference_params=c)
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        op(torch.zeros(2, 60, 8), inference_params=c)


def test_route_selection_boundary():
    import hyena_dna_b200 as H
    T = H.ops.EXTEND_FFT_MIN_N
    for t in (1, 1 << 14, 1 << 17, (1 << 20) - T):
        assert not H.ops.decode_extend_uses_fft(t, 1)
        assert not H.ops.decode_extend_uses_fft(t, T - 1)
        assert H.ops.decode_extend_uses_fft(t, T)
        assert H.ops.decode_extend_uses_fft(t, 8192)
