"""Left-padded prefill (``lengths``): the guards of hyena_b200_core_fwd_rows / hyena_b200_decode_hist_rows and the host
validation of HyenaOperator, Block, Backbone and DecodeCache, each firing before any device work (no GPU needed)."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")

P = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


def test_abi_present_and_no_new_kinds():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in ("hyena_b200_core_fwd_rows", "hyena_b200_decode_hist_rows"):
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header
    assert L.hyena_b200_abi_version() == 3 and L.hyena_b200_kind_count() == 33


def _core(p=P, sw=P, sb=P, kspec=P, fbias=P, y=P, rs=P, ib=None, c=None, gs=None, B=2, D=8, Lq=1024):
    return _lib.lib().hyena_b200_core_fwd_rows(p, ib, sw, sb, kspec, fbias, y, c, gs, rs, B, D, Lq, P, 1 << 30, None)


def _hist(p=P, h=P, tail=P, rs=P, ib=None, B=2, cache_B=2, order=2, Pn=16, Lcap=64):
    return _lib.lib().hyena_b200_decode_hist_rows(p, ib, P, P, h, tail, rs, B, cache_B, 8, order, Pn, Lcap, None)


def test_core_fwd_rows_guards():
    n0 = _lib.launch_count()
    odd, odd8 = ctypes.c_void_p(258), ctypes.c_void_p(260)
    for kw, msg in [(dict(rs=None), "null pointer"), (dict(p=None), "null pointer"), (dict(y=None), "null pointer"),
                    (dict(kspec=None), "null pointer"), (dict(B=0), "bad shape"), (dict(D=0), "bad shape"),
                    (dict(Lq=0), "bad shape"), (dict(Lq=(1 << 20) + 1), "exceeds the supported maximum"),
                    (dict(B=65536), "too large"), (dict(p=odd), "misaligned"), (dict(rs=odd), "misaligned"),
                    (dict(y=odd), "misaligned"), (dict(ib=odd), "misaligned"), (dict(c=odd), "misaligned"),
                    (dict(kspec=odd8), "misaligned"), (dict(gs=odd8), "misaligned")]:
        assert _core(**kw) != 0 and msg in _err(), (kw, _err())
    assert _lib.launch_count() == n0


def test_decode_hist_rows_guards():
    n0 = _lib.launch_count()
    odd = ctypes.c_void_p(258)
    for kw, msg in [(dict(rs=None), "null pointer"), (dict(p=None), "null pointer"), (dict(h=None), "null pointer"),
                    (dict(tail=None), "null pointer"), (dict(Pn=0), "outside"), (dict(Pn=65), "outside"),
                    (dict(cache_B=3), "differs"), (dict(order=1), "order"), (dict(Lcap=(1 << 20) + 1), "exceeds"),
                    (dict(B=0), "bad shape"), (dict(rs=odd), "misaligned"), (dict(h=odd), "misaligned"),
                    (dict(p=odd), "misaligned"), (dict(ib=odd), "misaligned")]:
        assert _hist(**kw) != 0 and msg in _err(), (kw, _err())
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- host side (device stubbed)
def _cpu_cache(op, B=3, lcap=64, t=0, seed=0):
    H = _H()
    g = torch.Generator().manual_seed(seed)
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    c = H.DecodeCache(op, B, lcap, lcap, torch.randn(F * ld + 4, generator=g), torch.randn(F, generator=g),
                      torch.zeros(O - 1, B, D, ld), torch.randn(B, C, 2, generator=g), torch.zeros(B, C),
                      torch.zeros(B, D, (lcap + 1023) // 1024))
    c.t = t
    return c


@pytest.fixture
def no_device(monkeypatch):
    """Every device entry point of the prefill fails the test if reached."""
    H = _H()
    for name in ("core_forward", "decode_hist", "proj_gemm", "add_layer_norm", "filter_spectrum", "decode_step_auto"):
        monkeypatch.setattr(H.ops, name, lambda *a, _n=name, **k: pytest.fail(f"device work ({_n}) before validation"))
    return H


BAD = [([5, 5], "2 entries"), ([5, 5, 5, 5], "4 entries"), ([5, 0, 5], r"outside \[1, 8\]"), ([5, 9, 5], r"outside \[1, 8\]"),
       ([5, -1, 5], r"outside \[1, 8\]"), ([5, 2.5, 5], "integers"), ([5, True, 5], "integers"), ("abc", "integers"),
       (torch.ones(3, 1, dtype=torch.long), "1-D"), (torch.tensor([1.0, 2.0, 3.0]), "1-D"), (None, None)]


@pytest.mark.parametrize("lengths,msg", BAD[:-1])
@pytest.mark.parametrize("order", [2, 3])
def test_lengths_are_validated_first(no_device, lengths, msg, order):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5, order=order)
    u = torch.zeros(3, 8, 8)
    n0 = H.launch_count()
    for call in (lambda: op.prefill(u, _cpu_cache(op), lengths=lengths),
                 lambda: op.extend(u, _cpu_cache(op), lengths=lengths),
                 lambda: op(u, inference_params=_cpu_cache(op), lengths=lengths)):
        with pytest.raises(H.HyenaB200Error, match=msg):
            call()
    with torch.no_grad():
        with pytest.raises(H.HyenaB200Error, match=msg):
            op(u, lengths=lengths)
    assert H.launch_count() == n0


def test_valid_lengths_reach_the_device_check(no_device):
    """Valid lengths pass the host checks: on the CPU the next thing that fails is the missing CUDA device."""
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    u = torch.zeros(3, 8, 8)
    for lengths in ([8, 1, 2], (3, 8, 8), torch.tensor([1, 1, 1], dtype=torch.int32)):
        with pytest.raises(H.HyenaB200Error, match="CUDA"):
            op.prefill(u, _cpu_cache(op), lengths=lengths)
        with torch.no_grad(), pytest.raises(H.HyenaB200Error, match="CUDA"):
            op(u, lengths=lengths)


def test_raises_listed_in_the_docs(no_device):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    u = torch.zeros(3, 8, 8)
    n0 = H.launch_count()
    c = _cpu_cache(op, t=9)
    with pytest.raises(H.HyenaB200Error, match="step takes no lengths"):
        op.step(u[:, :1], c, lengths=[1, 1, 1])
    with pytest.raises(H.HyenaB200Error, match="step takes no lengths"):
        op(u[:, :1], inference_params=c, lengths=[1, 1, 1])
    with pytest.raises(H.HyenaB200Error, match="holds history or is branched"):
        op.extend(u, c, lengths=[8, 8, 8])
    with pytest.raises(H.HyenaB200Error, match="holds history or is branched"):
        op(u, inference_params=c, lengths=[8, 8, 8])
    with pytest.raises(H.HyenaB200Error, match="fresh cache"):
        op.prefill(u, c, lengths=[8, 8, 8])
    br = _cpu_cache(op, t=9)
    br._branched = True
    with pytest.raises(H.HyenaB200Error, match="holds history or is branched"):
        op.extend(u, br, lengths=[8, 8, 8])
    # training: forward(lengths) with grad required points at right padding
    with pytest.raises(H.HyenaB200Error, match="pad them on the right"):
        op(u, lengths=[8, 8, 8])
    with torch.no_grad():
        with pytest.raises(H.HyenaB200Error, match="l_max"):
            op(torch.zeros(3, 65, 8), lengths=[1, 1, 1])
    assert H.launch_count() == n0


def test_block_and_backbone_validate_before_the_first_kernel(no_device):
    H = no_device
    mixer = partial(H.HyenaOperator, l_max=64, emb_dim=5)
    block = H.Block(8, mixer_cls=mixer)
    bb = H.Backbone(8, 2, mixer)
    u = torch.zeros(3, 8, 8)
    n0 = H.launch_count()
    bad = [5, 0, 5]
    with pytest.raises(H.HyenaB200Error, match="outside"):
        block.prefill(u, None, _cpu_cache(block.mixer), lengths=bad)
    with pytest.raises(H.HyenaB200Error, match="outside"):
        block.extend(u, None, _cpu_cache(block.mixer), lengths=bad)
    with torch.no_grad(), pytest.raises(H.HyenaB200Error, match="outside"):
        block(u, lengths=bad)
    with pytest.raises(H.HyenaB200Error, match="pad them on the right"):
        block(u, lengths=[8, 8, 8])
    stack = H.DecodeCache.stack([_cpu_cache(layer.mixer) for layer in bb.layers])
    with pytest.raises(H.HyenaB200Error, match="outside"):
        bb.prefill(u, stack, lengths=bad)
    with torch.no_grad(), pytest.raises(H.HyenaB200Error, match="outside"):
        bb(u, lengths=bad)
    busy = H.DecodeCache.stack([_cpu_cache(layer.mixer, t=4) for layer in bb.layers])
    with pytest.raises(H.HyenaB200Error, match="holds history"):
        bb.extend(u, busy, lengths=[8, 8, 8])
    assert H.launch_count() == n0


def test_cache_start_bookkeeping(monkeypatch):
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5, order=3)
    c = _cpu_cache(op, t=0)
    nbytes = c.nbytes
    assert c.start is None and c.start_dev is None and c.lengths == (0, 0, 0)
    assert nbytes == H.DecodeCache.layout_nbytes(3, 8, 3, 64)
    c.set_start([3, 0, 7])
    c.t = 10
    assert c.start == (3, 0, 7) and c.lengths == (7, 10, 3)
    assert c.start_dev.dtype == torch.int32 and c.start_dev.tolist() == [3, 0, 7]
    assert c.nbytes == nbytes + 12
    monkeypatch.setattr(H.ops, "_history_conv", lambda cache, ld, h, o, hist, L: torch.zeros(h.shape[0], 8, L))
    br = c.fork([2, 0, 2], horizon=8)
    assert br.start == (7, 3, 7) and br.lengths == (3, 7, 3) and br.start_dev.tolist() == [7, 3, 7]
    sel = br.select([1, 1, 0])
    assert sel.start == (3, 3, 7)
    plain = _cpu_cache(op, t=10).fork([1])
    assert plain.start is None and plain.lengths == (10,)
    stack = H.DecodeCache.stack([c, _cpu_cache(op, t=10)])
    assert stack.start == (3, 0, 7)
    with pytest.raises(H.HyenaB200Error, match="set by its layers"):
        stack.set_start([0, 0, 0])
