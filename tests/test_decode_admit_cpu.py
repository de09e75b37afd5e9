"""Continuous batching (HyenaOperator.admit, DecodeCache.release / compact, hyena_b200_decode_admit / _decode_shift;
DESIGN.md section 4.15) without a GPU: the C ABI guards, the two plan functions walked exhaustively, a model of the shift
kernel's tile order, the time-invariance identity on the fp64 oracle and the host checks, each before any device work."""
import ctypes
from functools import partial
from importlib import import_module

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O

_lib = import_module("hyena_dna_b200._lib")
ops = import_module("hyena_dna_b200.ops")

PTR = ctypes.c_void_p(256)        # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


# ---------------------------------------------------------------------------------------------- C ABI
def test_abi_present_and_no_new_kinds():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in ("hyena_b200_decode_admit", "hyena_b200_decode_shift"):
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header
    assert L.hyena_b200_abi_version() == 3 and L.hyena_b200_kind_count() == 33


def _admit(p=PTR, h=PTR, tail=PTR, rows=PTR, rs=None, ib=None, k=2, cache_B=4, order=2, Pn=16, t=32, Lcap=64):
    return _lib.lib().hyena_b200_decode_admit(p, ib, PTR, PTR, h, tail, rows, rs, k, cache_B, 8, order, Pn, t, Lcap, None)


def _shift(h=PTR, B=2, order=2, t=32, shift=-8, Lcap=64):
    return _lib.lib().hyena_b200_decode_shift(h, B, 8, order, t, shift, Lcap, None)


def test_decode_admit_guards():
    n0 = _lib.launch_count()
    odd = ctypes.c_void_p(258)
    for kw, msg in [(dict(p=None), "null pointer"), (dict(h=None), "null pointer"), (dict(tail=None), "null pointer"),
                    (dict(rows=None), "null pointer"), (dict(k=5), "5 prompts"), (dict(k=0), "bad shape"),
                    (dict(order=1), "order"), (dict(Lcap=(1 << 20) + 4, t=8), "exceeds"), (dict(Pn=33), "cannot end"),
                    (dict(Pn=0), "cannot end"), (dict(t=65), "outside the decode cache"), (dict(p=odd), "misaligned"),
                    (dict(h=odd), "misaligned"), (dict(rows=odd), "misaligned"), (dict(rs=odd), "misaligned"),
                    (dict(ib=odd), "misaligned")]:
        assert _admit(**kw) != 0 and msg in _err(), (kw, _err())
    assert _lib.launch_count() == n0


def test_decode_shift_guards():
    n0 = _lib.launch_count()
    for kw, msg in [(dict(h=None), "null pointer"), (dict(h=ctypes.c_void_p(264)), "16-byte aligned"),
                    (dict(shift=-6), "multiple of 4"), (dict(shift=2), "multiple of 4"), (dict(shift=-36), "left shift"),
                    (dict(shift=36), "right shift"), (dict(t=65), "outside"), (dict(B=0), "bad shape"),
                    (dict(order=32), "order")]:
        assert _shift(**kw) != 0 and msg in _err(), (kw, _err())
    assert _shift(shift=0) == 0                      # nothing to move: no launch
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- plans, exhaustively
WINDOWS = [(0, 0), (0, 4), (4, 8), (8, 4), (12, 16), (16, 3)]


def test_admit_plan_exhaustive():
    for lcap in range(1, 26):
        for t in range(0, lcap + 1):
            for P in range(1, lcap + 3):
                for wb, wc in WINDOWS:
                    if P > lcap:
                        with pytest.raises(_lib.HyenaB200Error, match="exceeds Lcap"):
                            ops.decode_admit_plan(t, lcap, P, wb, wc)
                        continue
                    need = (P - t + 3) // 4 * 4 if P > t > 0 else 0
                    if t + need > lcap:
                        with pytest.raises(_lib.HyenaB200Error, match="right shift"):
                            ops.decode_admit_plan(t, lcap, P, wb, wc)
                        continue
                    shift, t2, keep = ops.decode_admit_plan(t, lcap, P, wb, wc)
                    assert shift % 4 == 0 and shift >= 0
                    assert P <= t2 <= lcap
                    assert t2 == (P if t == 0 else t + shift)
                    assert shift < P - t + 4 if shift else True            # the least multiple of 4 that makes room
                    b2 = wb + shift
                    holds = wc > 0 and wb <= t < wb + wc and b2 <= t2 < b2 + wc and (b2 + wc <= lcap or not shift) and t > 0
                    assert keep == holds, (lcap, t, P, wb, wc)


def test_compact_plan_exhaustive():
    B = 3
    for t in range(0, 30):
        for starts in [(0,) * B] + [tuple(s) for s in np.ndindex(*(t + 1,) * B)][::max(1, t // 3)]:
            for free in ((), (0,), (1, 2), (0, 1, 2)):
                for wb, wc in WINDOWS:
                    shift, t2, keep = ops.decode_compact_plan(t, starts, free, wb, wc)
                    m = -shift
                    assert m % 4 == 0 and 0 <= m <= t and t2 == t - m
                    live = [s for b, s in enumerate(starts) if b not in free]
                    assert all(m <= s for s in live)                     # no live row loses a real position
                    want = min(live) if live else t
                    assert m == want - want % 4
                    b2 = wb - m
                    assert keep == (wc > 0 and b2 >= 0 and b2 <= t2 < b2 + wc), (t, starts, free, wb, wc)


# ---------------------------------------------------------------------------------------------- shift kernel tile order
def _shift_model(row, t, shift, threads, vec):
    """decode_shift_kernel on one row (numpy, float4 = 4 words), one barrier between each tile's loads and stores ->
    (row after the shift, the words a load read after an earlier store had overwritten them)."""
    h = row.reshape(-1, 4).copy()
    stored = np.zeros(h.shape[0], bool)
    stale = []
    n4, tile = (t + 3) // 4, threads * vec
    if shift < 0:
        m4 = -shift // 4
        w4 = n4 - m4
        for q0 in range(0, max(w4, 0), tile):
            qs = [q0 + u * threads + x for u in range(vec) for x in range(threads) if q0 + u * threads + x < w4]
            stale += [q + m4 for q in qs if stored[q + m4]]
            vals = {q: h[q + m4].copy() for q in qs}
            for q in qs:
                h[q], stored[q] = vals[q], True
    else:
        d4 = shift // 4
        for q1 in range(n4, 0, -tile):
            qs = [q1 - 1 - (u * threads + x) for u in range(vec) for x in range(threads) if q1 - 1 - (u * threads + x) >= 0]
            stale += [q for q in qs if stored[q]]
            vals = {q: h[q].copy() for q in qs}
            for q in qs:
                h[q + d4], stored[q + d4] = vals[q], True
        h[:d4] = 0.0
    return h.reshape(-1), stale


@pytest.mark.parametrize("direction", ["left", "right"])
def test_shift_tile_order_never_reads_a_stored_word(direction):
    threads, vec = 4, 2                                   # a tile of 8 float4s = 32 positions
    tile = 4 * threads * vec
    rng = np.random.default_rng(0)
    for ld in (64, 68, 128, 132):
        for t in (1, 3, 4, 31, 32, 33, 63, ld - 4, ld):
            if t > ld:
                continue
            ms = {4, tile - 4, tile, tile + 4, 2 * tile, t - t % 4} if direction == "left" else \
                 {4, tile - 4, tile, tile + 4, 2 * tile, ld - (t + 3) // 4 * 4}
            for m in sorted(x for x in ms if x > 0):
                if direction == "left" and m > t:
                    continue
                if direction == "right" and (t + 3) // 4 * 4 + m > ld:
                    continue
                row = rng.standard_normal(ld).astype(np.float32)
                got, stale = _shift_model(row, t, -m if direction == "left" else m, threads, vec)
                assert not stale, (ld, t, m, stale)
                want = row.copy()
                T4 = (t + 3) // 4 * 4
                if direction == "left":
                    want[:T4 - m] = row[m:T4]
                else:
                    want[m:T4 + m] = row[:T4]
                    want[:m] = 0.0
                assert np.array_equal(got, want), (ld, t, m)


# ---------------------------------------------------------------------------------------------- time invariance (oracle)
def _masked_operator(u, P, off):
    """y_pre of the operator in fp64 over positions with every input before ``off`` masked as a prefill's pads are: the
    in_proj output (with its bias) and every g zeroed there; direct-sum convolutions (fixed order per output)."""
    B, L, D = u.shape
    order = P["in_proj.weight"].shape[0] // D - 1
    keep = (torch.arange(L) >= off)[None, None, :]
    p = torch.where(keep, F.linear(u, P["in_proj.weight"], P["in_proj.bias"]).transpose(1, 2), 0.0)
    uc = O.short_filter(p, P["short_filter.weight"], P["short_filter.bias"], L)
    *x, v = uc.split(D, dim=1)
    k = O.hyena_filter(L, P)[0].transpose(0, 1).reshape(D, order - 1, L)
    bias = P["filter_fn.bias"].reshape(D, order - 1)
    for o, x_i in enumerate(reversed(x[1:])):
        g = torch.where(keep, v * x_i, 0.0)
        v = O.fftconv_direct(g, k[:, o], bias[:, o])
    return torch.where(keep, v * x[0], 0.0)


@pytest.mark.parametrize("order", [2, 3])
def test_zero_prefixed_row_decodes_like_the_unpadded_row(order):
    """A prompt placed at any offset with a zero history before it gives, at every later position, the bits of the
    unpadded prompt (fp64, direct sums): the identity admission rests on."""
    D, n = 4, 24
    g = torch.Generator().manual_seed(order)
    P = O.to_dtype(O.init_params(D, 128, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.1), torch.float64)
    P["in_proj.bias"] = 0.1 * torch.randn(P["in_proj.bias"].shape, generator=g, dtype=torch.float64)
    u = torch.randn(1, n, D, generator=g, dtype=torch.float64)
    ref = _masked_operator(u, P, 0)
    for off in (1, 2, 3, 4, 5, 17, 40):
        junk = 5.0 * torch.randn(1, off, D, generator=g, dtype=torch.float64)
        y = _masked_operator(torch.cat([junk, u], 1), P, off)
        assert torch.equal(y[..., off:], ref), off
        assert not y[..., :off].any()


# ---------------------------------------------------------------------------------------------- host checks first
def _cpu_cache(op, B=4, lcap=64, t=0, seed=0):
    H = _H()
    g = torch.Generator().manual_seed(seed)
    ld = (lcap + 3) // 4 * 4
    D, Od = op.d_model, op.order
    Fc, C = (Od - 1) * D, (Od + 1) * D
    c = H.DecodeCache(op, B, lcap, lcap, torch.randn(Fc * ld + 4, generator=g), torch.randn(Fc, generator=g),
                      torch.zeros(Od - 1, B, D, ld), torch.randn(B, C, 2, generator=g), torch.zeros(B, C),
                      torch.zeros(B, D, (lcap + 1023) // 1024))
    c.t = t
    return c


@pytest.fixture
def no_device(monkeypatch):
    """Every device entry point of an admission fails the test if reached."""
    H = _H()
    for name in ("core_forward", "decode_hist", "decode_admit", "decode_shift", "proj_gemm", "add_layer_norm",
                 "filter_spectrum", "decode_step_auto"):
        monkeypatch.setattr(H.ops, name, lambda *a, _n=name, **k: pytest.fail(f"device work ({_n}) before validation"))
    return H


CASES = [(dict(rows=[0, 4]), r"rows 4 outside \[0, 4\)"), (dict(rows=[1, 1]), "repeat"), (dict(rows=[0]), "1 rows for 2"),
         (dict(rows=[]), "empty"), (dict(rows=[0.5, 1]), "integers"), (dict(P=65), "exceeds Lcap"),
         (dict(t=41, P=63), "right shift"), (dict(lengths=[3, 0]), "outside"), (dict(lengths=[3]), "1 entries"),
         (dict(lengths=[9, 1]), "outside"), (dict(grad=True), "requires grad"), (dict(branched=True), "branched"),
         (dict(shape=(2, 8, 5)), "prompts must be")]


@pytest.mark.parametrize("case,msg", CASES)
@pytest.mark.parametrize("order", [2, 3])
def test_admit_checks_run_before_device_work(no_device, case, msg, order):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5, order=order)
    mixer = partial(H.HyenaOperator, l_max=64, emb_dim=5, order=order)
    block, bb = H.Block(8, mixer_cls=mixer), H.Backbone(8, 2, mixer)
    P, t = case.get("P", 8), case.get("t", 20)
    u = torch.zeros(case.get("shape", (2, P, 8)), requires_grad=case.get("grad", False))
    rows, lengths = case.get("rows", [3, 1]), case.get("lengths")

    def cache(m):
        c = _cpu_cache(m, t=t)
        c._branched = case.get("branched", False)
        return c
    n0 = H.launch_count()
    for call in (lambda: op.admit(u, cache(op), rows, lengths),
                 lambda: block.admit(u, None, cache(block.mixer), rows, lengths),
                 lambda: bb.admit(u, H.DecodeCache.stack([cache(layer.mixer) for layer in bb.layers]), rows, lengths)):
        with pytest.raises(H.HyenaB200Error, match=msg):
            call()
    assert H.launch_count() == n0


def test_valid_admission_reaches_the_device_check(no_device):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    for t, P, lengths in ((20, 8, None), (0, 8, [8, 3]), (3, 60, [1, 60]), (64, 64, None)):
        with pytest.raises(H.HyenaB200Error, match="CUDA"):
            op.admit(torch.zeros(2, P, 8), _cpu_cache(op, t=t), torch.tensor([2, 0]), lengths)


def test_release_and_compact_bookkeeping(no_device, monkeypatch):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op, t=30)
    nbytes = c.nbytes
    c.set_start([13, 0, 22, 9])
    c.release([1])
    assert c.free == frozenset({1}) and c.lengths == (17, 0, 8, 21)
    c.release(torch.tensor([3]))
    assert c.free == frozenset({1, 3}) and c.lengths == (17, 0, 8, 0)
    with pytest.raises(H.HyenaB200Error, match="outside"):
        c.release([4])
    shifts = []
    monkeypatch.setattr(H.ops, "decode_shift", lambda cache, s: (shifts.append(s), setattr(cache, "t", cache.t + s),
                                                                 cache.set_start([max(x + s, 0) for x in cache.start])))
    c.win_b, c.win_wc = 16, 32
    assert c.compact() == 12 and shifts == [-12] and c.t == 18 and c.win_wc == 32
    assert c.lengths == (17, 0, 8, 0)
    c.win_b = 8
    c.set_start([13, 0, 30, 9])                       # m = 12 > win_b: the window closes
    c.t = 30
    assert c.compact() == 12 and (c.win_b, c.win_wc) == (0, 0)
    assert H.DecodeCache.layout_nbytes(4, 8, 2, 64) == nbytes
    stack = H.DecodeCache.stack([_cpu_cache(op, t=12), _cpu_cache(op, t=12)])
    stack.release([0, 2])
    assert all(layer.free == frozenset({0, 2}) for layer in stack.layers) and stack.lengths == (0, 12, 0, 12)
    br = _cpu_cache(op, t=9)
    br._branched = True
    for call in (lambda: br.release([0]), br.compact):
        with pytest.raises(H.HyenaB200Error, match="branched"):
            call()
