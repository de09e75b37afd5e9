"""A 16-bit decode history without a GPU: dtype validation, the cache's byte counts and the C guards of the _h16 entry
points (DESIGN.md section 4.16).  Every call below is rejected before any CUDA work, as in tests/test_abi_errors_cpu.py."""
import ctypes
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")
HALF = [torch.float16, torch.bfloat16]
CODES = {torch.float16: 1, torch.bfloat16: 2}
PTR = ctypes.c_void_p(1 << 20)       # 16-byte aligned, never dereferenced
ODD2 = ctypes.c_void_p((1 << 20) + 2)    # 2-byte aligned: one fp16 element, not four
ODD1 = ctypes.c_void_p((1 << 20) + 1)


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


def _op(D=8, L=64, order=2):
    return _H().HyenaOperator(D, L, order=order, emb_dim=5, w=10.0)


# ------------------------------------------------------------------------------------------ host validation
@pytest.mark.parametrize("bad", [torch.float64, torch.int8, torch.float8_e4m3fn, "float16", None, torch.complex64])
def test_history_dtype_is_validated_before_allocation(bad):
    H = _H()
    op = _op()
    with pytest.raises(H.HyenaB200Error, match="history_dtype"):
        op.allocate_decode_cache(1, 16, history_dtype=bad)        # the dtype check comes before the CUDA check
    with pytest.raises(H.HyenaB200Error, match="history_dtype"):
        H.DecodeCache.allocate(op, 1, 16, history_dtype=bad)
    with pytest.raises(H.HyenaB200Error, match="history_dtype"):
        H.DecodeCache.layout_nbytes(1, 8, 2, 16, history_dtype=bad)
    mixer = lambda dim: _op(dim)
    m = H.Backbone(8, 2, mixer)
    with pytest.raises(H.HyenaB200Error, match="history_dtype"):
        m.allocate_decode_cache(1, 16, history_dtype=bad)


@pytest.mark.parametrize("dtype", [torch.float32] + HALF)
def test_cpu_operator_still_refused(dtype):
    """A valid dtype passes the dtype check and then meets the usual CUDA-only refusal on a CPU operator."""
    H = _H()
    with pytest.raises(H.HyenaB200Error, match="CUDA"):
        _op().allocate_decode_cache(1, 16, history_dtype=dtype)


# ------------------------------------------------------------------------------------------ byte counts
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("B,D,order,lcap", [(1, 256, 2, 1 << 20), (64, 256, 2, 1 << 17), (3, 100, 3, 1021), (2, 1, 4, 5)])
def test_layout_nbytes(dtype, B, D, order, lcap):
    H = _H()
    ld, F, C = (lcap + 3) // 4 * 4, (order - 1) * D, (order + 1) * D
    hist = (order - 1) * B * D * ld
    rest = 4 * ((F * ld + 4) + F + B * C * 2 + B * C + B * D * -(-lcap // 1024))
    assert H.DecodeCache.layout_nbytes(B, D, order, lcap) == rest + 4 * hist              # the default is unchanged
    assert H.DecodeCache.layout_nbytes(B, D, order, lcap, torch.float32) == rest + 4 * hist
    assert H.DecodeCache.layout_nbytes(B, D, order, lcap, dtype) == rest + 2 * hist
    assert H.DecodeCache.layout_nbytes(B, D, order, lcap, history_dtype=dtype) == rest + 2 * hist


@pytest.mark.parametrize("dtype", HALF)
def test_nbytes_reports_the_smaller_history(dtype):
    """A cache built from host tensors of the allocated layout: nbytes counts h at two bytes per element, and a stack
    reports the history dtype of its layers."""
    H = _H()
    B, D, order, lcap = 3, 5, 3, 37
    ld, F, C = (lcap + 3) // 4 * 4, (order - 1) * D, (order + 1) * D

    def cache(hd):
        f32 = dict(dtype=torch.float32)
        c = H.DecodeCache(None, B, lcap, lcap, torch.zeros(F * ld + 4, **f32), torch.zeros(F, **f32),
                          torch.zeros(order - 1, B, D, ld, dtype=hd), torch.zeros(B, C, 2, **f32), torch.zeros(B, C, **f32),
                          torch.zeros(B, D, 1, **f32))
        return c
    c16, c32 = cache(dtype), cache(torch.float32)
    assert c16.history_dtype == dtype and c32.history_dtype == torch.float32
    assert c32.nbytes == H.DecodeCache.layout_nbytes(B, D, order, lcap)
    assert c16.nbytes == H.DecodeCache.layout_nbytes(B, D, order, lcap, dtype)
    assert c32.nbytes - c16.nbytes == 2 * (order - 1) * B * D * ld
    st = H.DecodeCache.stack([cache(dtype), cache(dtype)])
    assert st.history_dtype == dtype and st.nbytes == 2 * c16.nbytes


# ------------------------------------------------------------------------------------------ C guards of the _h16 entries
def _call(name, code, **kw):
    """hyena_b200_decode_<name>_h16 with valid arguments (B = 2, D = 8, order 2, Lcap 64), overridden by kw."""
    L = _lib.lib()
    a = dict(p=PTR, ib=None, sw=PTR, sb=PTR, k=PTR, fb=PTR, h=PTR, tail=PTR, s=PTR, v=None, out=PTR, part=PTR, win=PTR,
             f=PTR, parent=PTR, rows=PTR, rs=PTR, pos=PTR, B=2, D=8, order=2, o=0, t=32, n=4, b=32, Wc=16, W=16, Hc=16,
             H=16, Lcap=64, P=16, shift=-8, groups=None)
    a.update(kw)
    g = a["groups"] if a["groups"] is not None else L.hyena_b200_decode_extend_groups(a["B"], a["D"], a["t"], a["n"])
    fn = getattr(L, f"hyena_b200_decode_{name}_h16")
    args = {
        "hist": (a["p"], a["ib"], a["sw"], a["sb"], a["h"], a["tail"], a["B"], a["B"], a["D"], a["order"], a["P"], a["Lcap"]),
        "hist_rows": (a["p"], a["ib"], a["sw"], a["sb"], a["h"], a["tail"], a["rs"], a["B"], a["B"], a["D"], a["order"],
                      a["P"], a["Lcap"]),
        "admit": (a["p"], a["ib"], a["sw"], a["sb"], a["h"], a["tail"], a["rows"], None, 1, a["B"], a["D"], a["order"],
                  a["P"], a["t"], a["Lcap"]),
        "shift": (a["h"], a["B"], a["D"], a["order"], a["t"], a["shift"], a["Lcap"]),
        "step": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"], a["part"],
                 a["B"], a["B"], a["D"], a["order"], a["o"], a["t"], a["Lcap"]),
        "win_step": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"],
                     a["part"], a["win"], a["B"], a["B"], a["D"], a["order"], a["o"], a["t"], a["b"], a["Wc"], a["W"],
                     a["Lcap"]),
        "extend_hist": (a["p"], a["ib"], a["sw"], a["sb"], a["h"], a["tail"], a["s"], a["B"], a["B"], a["D"], a["order"],
                        a["t"], a["n"], a["Lcap"]),
        "extend_dot": (a["h"], a["k"], a["part"], g, a["B"], a["B"], a["D"], a["order"], a["o"], a["t"], a["n"], a["Lcap"]),
        "extend_combine": (a["part"], a["n"], 1, 1, a["fb"], a["h"], a["s"], a["out"], a["B"], a["B"], a["D"], a["order"],
                           a["o"], a["t"], a["n"], a["Lcap"]),
        "branch_step": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"],
                        a["part"], a["f"], a["parent"], a["B"], a["D"], a["order"], a["o"], a["t"], a["b"], a["Hc"],
                        a["H"], a["Lcap"]),
        "branch_extend_hist": (a["p"], a["ib"], a["sw"], a["sb"], a["h"], a["tail"], a["s"], a["B"], a["D"], a["order"],
                               a["t"], a["n"], a["b"], a["Hc"], a["H"], a["Lcap"]),
        "branch_extend_dot": (a["h"], a["k"], a["part"], g, a["B"], a["D"], a["order"], a["o"], a["t"], a["n"], a["b"],
                              a["Hc"], a["H"], a["Lcap"]),
        "branch_combine": (a["part"], a["n"], 1, 1, a["fb"], a["h"], a["s"], a["out"], a["f"], a["parent"], a["B"], a["D"],
                           a["order"], a["o"], a["t"], a["n"], a["b"], a["Hc"], a["H"], a["Lcap"]),
        "step_dev": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"],
                     a["part"], a["pos"], a["B"], a["B"], a["D"], a["order"], a["o"], a["t"], a["Lcap"]),
        "win_step_dev": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"],
                         a["part"], a["win"], a["pos"], a["B"], a["B"], a["D"], a["order"], a["o"], a["W"], a["Lcap"]),
        "branch_step_dev": (a["p"], a["ib"], a["sw"], a["sb"], a["k"], a["fb"], a["h"], a["tail"], a["s"], a["v"], a["out"],
                            a["part"], a["f"], a["parent"], a["pos"], a["B"], a["D"], a["order"], a["o"], a["H"], a["Lcap"]),
    }[name]
    return fn(code, *args, None)


NAMES = ["hist", "hist_rows", "admit", "shift", "step", "win_step", "extend_hist", "extend_dot", "extend_combine",
         "branch_step", "branch_extend_hist", "branch_extend_dot", "branch_combine", "step_dev", "win_step_dev",
         "branch_step_dev"]
# entry points whose fp32 twin checks h's alignment (16 bytes, or 4 for the hist_rows / admit element writes)
VEC_ALIGNED = ["shift", "step", "win_step", "extend_dot", "branch_step", "branch_extend_dot", "step_dev", "win_step_dev",
               "branch_step_dev"]
ELEM_ALIGNED = ["hist_rows", "admit", "extend_combine", "branch_combine"]


def test_every_h16_entry_point_is_bound():
    L = _lib.lib()
    for n in NAMES:
        assert hasattr(L, f"hyena_b200_decode_{n}_h16")
        assert _lib.SIGNATURES[f"hyena_b200_decode_{n}_h16"][1] == [ctypes.c_int] + _lib.SIGNATURES[f"hyena_b200_decode_{n}"][1]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("code", [0, 3, -1, 16, 1 << 30])
def test_unknown_dtype_code(name, code):
    n0 = _lib.launch_count()
    assert _call(name, code) != 0 and "unknown history dtype code" in _err(), _err()
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dtype", HALF)
def test_null_history(name, dtype):
    n0 = _lib.launch_count()
    assert _call(name, CODES[dtype], h=None) != 0 and "null pointer" in _err(), _err()
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("dtype", HALF)
def test_history_alignment(dtype):
    """A 16-bit history needs 4-element (8-byte) alignment where the vector loads and the shift read it, 2-byte
    alignment where single elements are written; 8-byte alignment is enough (half of the fp32 twin's 16)."""
    n0 = _lib.launch_count()
    code = CODES[dtype]
    for name in VEC_ALIGNED:
        assert _call(name, code, h=ODD2) != 0 and "8-byte aligned" in _err(), (name, _err())
    for name in ELEM_ALIGNED:
        assert _call(name, code, h=ODD1) != 0 and "aligned" in _err(), (name, _err())
    for name in ["extend_combine", "branch_combine"]:          # out is the next recurrence's 16-bit history there
        assert _call(name, code, order=3, out=ODD1) != 0 and "aligned" in _err(), (name, _err())
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("dtype", HALF)
def test_ranges_are_checked(dtype):
    n0 = _lib.launch_count()
    code = CODES[dtype]
    cases = [("hist", dict(P=65), "outside"), ("hist", dict(order=1), "order"), ("hist", dict(Lcap=(1 << 20) + 4), "exceeds"),
             ("admit", dict(P=33), "cannot end"), ("shift", dict(shift=-6), "multiple of 4"),
             ("shift", dict(shift=36), "right shift"), ("step", dict(t=64), "outside the decode cache"),
             ("step", dict(o=1), "recurrence"), ("win_step", dict(t=31), "outside the window"),
             ("extend_hist", dict(n=0), "n must be"), ("extend_dot", dict(t=61), "outside the decode cache"),
             ("extend_dot", dict(groups=7), "partials sized"), ("extend_combine", dict(o=2), "recurrence"),
             ("branch_step", dict(b=30), "branch base"), ("branch_extend_dot", dict(H=14), "branch history width"),
             ("branch_combine", dict(t=48), "branch horizon"), ("step_dev", dict(t=65), "position bound"),
             ("win_step_dev", dict(W=0), "window width"), ("branch_step_dev", dict(H=6), "branch history width"),
             ("step_dev", dict(pos=None), "device position")]
    for name, kw, msg in cases:
        assert _call(name, code, **kw) != 0 and msg in _err(), (name, kw, _err())
    assert _lib.launch_count() == n0
