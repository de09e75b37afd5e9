"""Incremental decoding: argument checks of the C ABI and of the Python API, and the cache layout (no GPU needed: every
call below is rejected before any CUDA work)."""
import ctypes
import types
from functools import partial
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


P = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _step(p_t=P, k=P, h=P, tail=P, v_in=None, B=1, cache_B=1, D=8, order=2, o=0, t=0, Lcap=64):
    return _lib.lib().hyena_b200_decode_step(p_t, P, P, P, k, P, h, tail, P, v_in, P, P, B, cache_B, D, order, o, t, Lcap, None)


def test_decode_step_abi_guards():
    assert _step(k=None) != 0 and "null pointer" in _err()
    assert _step(h=None) != 0 and "null pointer" in _err()
    assert _step(p_t=None) != 0 and "null pointer" in _err()
    assert _step(order=3, o=1) != 0 and "v_in" in _err()                    # a later recurrence needs the previous output
    assert _step(t=64, Lcap=64) != 0 and "outside the decode cache" in _err()
    assert _step(t=-1) != 0 and "outside the decode cache" in _err()
    assert _step(B=2, cache_B=1) != 0 and "differs from the decode cache" in _err()
    assert _step(o=1) != 0 and "recurrence" in _err()
    assert _step(order=1) != 0 and "order" in _err()
    assert _step(Lcap=(1 << 20) + 1) != 0 and "exceeds the supported maximum" in _err()


def test_decode_hist_abi_guards():
    L = _lib.lib()
    hist = lambda p=P, B=1, cache_B=1, Pn=16, Lcap=64: L.hyena_b200_decode_hist(p, P, P, P, P, P, B, cache_B, 8, 2, Pn, Lcap, None)
    assert hist(p=None) != 0 and "null pointer" in _err()
    assert hist(Pn=65) != 0 and "prefill of 65 positions" in _err()
    assert hist(Pn=0) != 0 and "prefill of 0 positions" in _err()
    assert hist(B=3, cache_B=2) != 0 and "differs from the decode cache" in _err()


def test_profiler_kinds_include_decoding():
    L = _lib.lib()
    names = [L.hyena_b200_kind_name(i).decode() for i in range(L.hyena_b200_kind_count())]
    assert "decode_hist" in names and "decode_step" in names
    assert L.hyena_b200_abi_version() == 3


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


def test_nbytes_matches_the_layout():
    import hyena_dna_b200 as H
    for B, D, O, lcap in [(1, 256, 2, 1 << 20), (2, 64, 2, 1041), (3, 8, 3, 64), (1, 16, 4, 4097)]:
        ld = -(-lcap // 4) * 4
        F, C = (O - 1) * D, (O + 1) * D
        want = 4 * (F * ld + 4 + F + (O - 1) * B * D * ld + 2 * B * C + B * C + B * D * -(-lcap // 1024))
        assert H.DecodeCache.layout_nbytes(B, D, O, lcap) == want
    op = _op(order=3)
    c = _cpu_cache(op, B=2, lcap=50)
    assert c.nbytes == H.DecodeCache.layout_nbytes(2, 8, 3, 50)
    stack = H.DecodeCache.stack([c, _cpu_cache(_op(), B=2, lcap=50)])
    assert stack.nbytes == c.nbytes + H.DecodeCache.layout_nbytes(2, 8, 2, 50)


def test_api_guards():
    import hyena_dna_b200 as H
    op = _op()
    c = _cpu_cache(op)
    u = torch.zeros(2, 1, 8)
    with pytest.raises(H.HyenaB200Error, match="requires grad"):
        op.step(u.clone().requires_grad_(True), c)
    with pytest.raises(H.HyenaB200Error, match="CUDA"):              # everything else is valid: the CPU tensor is the fault
        op.step(u, c)
    with pytest.raises(H.HyenaB200Error, match="batch size 3"):
        op.step(torch.zeros(3, 1, 8), c)
    with pytest.raises(H.HyenaB200Error, match=r"\(B, 1, 8\)"):
        op.step(torch.zeros(2, 2, 8), c)
    with pytest.raises(H.HyenaB200Error, match="DecodeCache"):
        op.step(u, {"not": "a cache"})
    with pytest.raises(H.HyenaB200Error, match="not allocated for this"):
        _op().step(u, c)
    c.t = 64                                                           # Lcap = l_max = 64: no position left
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        op.step(u, c)
    with pytest.raises(H.HyenaB200Error, match="fresh cache"):
        c.t = 3
        op.prefill(torch.zeros(2, 4, 8), c)
    c.t = 0
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        op.prefill(torch.zeros(2, 65, 8), c)
    with pytest.raises(H.HyenaB200Error, match="CUDA"):               # allocation on the CPU
        op.allocate_decode_cache(2, 64)


def test_bidirectional_filter_is_rejected():
    import hyena_dna_b200 as H
    op = _op(bidirectional=True)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        op.allocate_decode_cache(1, 16)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        op.step(torch.zeros(2, 1, 8), _cpu_cache(op))


def test_block_and_backbone_guards():
    import hyena_dna_b200 as H
    m = H.Backbone(8, 2, partial(H.HyenaOperator, l_max=64, emb_dim=5))
    with pytest.raises(H.HyenaB200Error, match="requires grad"):
        m.step(torch.zeros(1, 1, 8, requires_grad=True), None)
    with pytest.raises(H.HyenaB200Error, match="CUDA"):
        m.allocate_decode_cache(1, 64)


def test_other_inference_params_are_ignored():
    """Only a DecodeCache switches forward to decoding; anything else takes the ordinary path (here: the CPU error of
    forward itself, not a decoding error)."""
    import hyena_dna_b200 as H
    op = _op()
    u = torch.zeros(2, 4, 8)
    for ip in (None, object(), types.SimpleNamespace(max_seqlen=64, batch_size_offset=0, seqlen_offset=0)):
        with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
            op(u, inference_params=ip)
