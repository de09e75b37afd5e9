"""Packed variable-length batches (``cu_seqlens=``; DESIGN.md section 4.18) without a GPU: the bucket plan, the guards of
the three C entry points, the host validation of HyenaOperator, Block and Backbone, each firing before any device work,
and a self-check that the per-sequence truth the GPU tests use rejects leaky results."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU

_lib = import_module("hyena_dna_b200._lib")
ops = import_module("hyena_dna_b200.ops")

PTR = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


# ---------------------------------------------------------------------------------------------- helpers of the GPU tests
def packed_input(lengths, D, seed=0):
    """u (total, D) on the CPU with the sequences of ``lengths`` packed back to back, and cu (N+1 host integers)."""
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    u = O.nucleotide_activations(1, max(cu[-1], 1), D, seed=2222 + seed)[0][0, :cu[-1]]
    return u.contiguous(), cu


def seq_truth(u, dy, cu, P, dtype, device=None, only=None):
    """Truth of packed sequences: the oracle (O.operator_fwd_bwd) on each sequence alone in ``dtype`` on ``device`` (the
    sequences of one length run as one batch) -> ({i: y_i}, {i: du_i}, parameter gradients summed over the sequences).
    ``only``: the set of sequences to run (the others are left out of the sums)."""
    device = device or torch.device("cpu")
    Q = {k: v.to(device, dtype) for k, v in P.items()}
    by_len = {}
    for i, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        if b > a and (only is None or i in only):
            by_len.setdefault(b - a, []).append(i)
    ys, dus, sums = {}, {}, {}
    for n, seqs in by_len.items():
        uu = torch.stack([u[cu[i]:cu[i] + n] for i in seqs]).to(device, dtype)
        dd = torch.stack([dy[cu[i]:cu[i] + n] for i in seqs]).to(device, dtype)
        y, du, g = O.operator_fwd_bwd(uu, Q, dd)
        for j, i in enumerate(seqs):
            ys[i], dus[i] = y[j], du[j]
        for k, v in g.items():
            sums[k] = sums.get(k, 0) + v
    return ys, dus, sums


# ---------------------------------------------------------------------------------------------- bucket plan
def test_bucket_length():
    for n, L in [(1, 1024), (2, 1024), (3, 1024), (1023, 1024), (1024, 1024), (1025, 2048), (2048, 2048),
                 (2049, 4096), ((1 << 20) - 1, 1 << 20), (1 << 20, 1 << 20)]:
        assert ops.bucket_length(n) == L, n
        assert ops.bucket_length(n) == _lib.lib().hyena_b200_spectrum_elems(n)


def test_plan_rows_and_starts():
    lengths = [3, 0, 1024, 1, 1025, 2, 0, 1 << 20, 1023]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    plan = ops.packed_plan(cu)
    assert [b.L for b in plan] == [1024, 2048, 1 << 20]
    assert [b.seqs for b in plan] == [[0, 2, 3, 5, 8], [4], [7]]
    seen = []
    for b in plan:
        for i, sb, rs in zip(b.seqs, b.seg_base, b.row_start):
            n = cu[i + 1] - cu[i]
            assert rs == b.L - n and sb == cu[i + 1] - b.L and sb + rs == cu[i]
            seen.append(i)
    assert sorted(seen) == [0, 2, 3, 4, 5, 7, 8]               # zero-length sequences are skipped
    assert [b.offset for b in plan] == [0, 5, 6]


def test_plan_bucket_depends_on_own_length_only():
    """A sequence's row length and start are the same whatever its neighbours and its place."""
    g = torch.Generator().manual_seed(0)
    for _ in range(20):
        lengths = torch.randint(0, 5000, (30,), generator=g).tolist()
        lengths[7] = 1500
        perm = torch.randperm(30, generator=g).tolist()
        for ls in (lengths, [lengths[i] for i in perm]):
            cu = [0]
            for n in ls:
                cu.append(cu[-1] + n)
            i = ls.index(1500)
            rows = [(b.L, rs) for b in ops.packed_plan(cu) for s, rs in zip(b.seqs, b.row_start) if s == i]
            assert rows == [(2048, 548)]


def test_plan_splits_large_buckets():
    cu = list(range(ops.MAX_BUCKET_ROWS + 11))
    plan = ops.packed_plan(cu)
    assert [len(b.seqs) for b in plan] == [ops.MAX_BUCKET_ROWS, 10]
    assert plan[1].offset == ops.MAX_BUCKET_ROWS


# ---------------------------------------------------------------------------------------------- C entry points
def test_abi_present_and_no_new_kinds():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in ("hyena_b200_core_fwd_packed", "hyena_b200_core_bwd_packed", "hyena_b200_short_bwd_packed"):
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header
    assert L.hyena_b200_abi_version() == 3 and L.hyena_b200_kind_count() == 33


ODD, ODD8 = ctypes.c_void_p(258), ctypes.c_void_p(260)
SHAPE = [(dict(B=0), "bad shape"), (dict(D=0), "bad shape"), (dict(Lq=0), "bad shape"),
         (dict(Lq=(1 << 20) + 1), "exceeds the supported maximum"), (dict(B=65536), "too large"),
         (dict(total=0), "bad packed length"), (dict(sg=None), "null pointer"), (dict(rs=None), "null pointer"),
         (dict(sg=ODD8), "misaligned"), (dict(rs=ODD), "misaligned")]


def _fwd(p=PTR, kspec=PTR, y=PTR, c=None, gs=None, ib=None, sg=PTR, rs=PTR, total=5000, B=2, D=8, Lq=1024):
    return _lib.lib().hyena_b200_core_fwd_packed(p, ib, PTR, PTR, kspec, PTR, y, c, gs, sg, rs, total, B, D, Lq, PTR,
                                                 1 << 30, None)


def _bwd(dy=PTR, p=PTR, kspec=PTR, c=PTR, dk=PTR, ds=PTR, gs=None, ib=None, sg=PTR, rs=PTR, total=5000, B=2, D=8,
         Lq=1024):
    return _lib.lib().hyena_b200_core_bwd_packed(dy, p, ib, PTR, PTR, kspec, PTR, c, gs, dk, PTR, PTR, PTR, ds, sg, rs,
                                                 total, B, D, Lq, PTR, 1 << 30, None)


def _short(ds=PTR, dp=PTR, dib=None, sg=PTR, rs=PTR, total=5000, B=2, D=24, Lq=1024):
    return _lib.lib().hyena_b200_short_bwd_packed(ds, PTR, dp, dib, sg, rs, total, B, D, Lq, None)


@pytest.mark.parametrize("fn,cases", [
    (_fwd, SHAPE + [(dict(p=None), "null pointer"), (dict(y=None), "null pointer"), (dict(kspec=None), "null pointer"),
                    (dict(p=ODD), "misaligned"), (dict(y=ODD), "misaligned"), (dict(c=ODD), "misaligned"),
                    (dict(ib=ODD), "misaligned"), (dict(kspec=ODD8), "misaligned"), (dict(gs=ODD8), "misaligned")]),
    (_bwd, SHAPE + [(dict(dy=None), "null pointer"), (dict(c=None), "null pointer"), (dict(dk=None), "null pointer"),
                    (dict(ds=None), "null pointer"), (dict(dy=ODD), "misaligned"), (dict(ds=ODD), "misaligned"),
                    (dict(c=ODD), "misaligned"), (dict(kspec=ODD8), "misaligned"), (dict(gs=ODD8), "misaligned")]),
    (_short, SHAPE + [(dict(ds=None), "null pointer"), (dict(dp=None), "null pointer"), (dict(ds=ODD), "misaligned"),
                      (dict(dp=ODD), "misaligned"), (dict(dib=ODD), "misaligned")]),
], ids=["core_fwd_packed", "core_bwd_packed", "short_bwd_packed"])
def test_packed_entry_point_guards(fn, cases):
    n0 = _lib.launch_count()
    for kw, msg in cases:
        if fn is _short and "D" in kw:
            continue
        assert fn(**kw) != 0 and msg in _err(), (fn.__name__, kw, _err())
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- host validation
def _op(**kw):
    H = _H()
    return H.HyenaOperator(8, 4096, emb_dim=5, **kw)


@pytest.mark.parametrize("cu,msg", [
    (torch.tensor([1, 3, 10]), "cu_seqlens[0] must be 0"),
    (torch.tensor([0, 5, 3, 10]), "non-decreasing"),
    (torch.tensor([0, 3, 9]), "must equal the number of packed positions"),
    (torch.tensor([0, 3, 11]), "must equal the number of packed positions"),
    (torch.tensor([0.0, 10.0]), "integer"),
    (torch.tensor([True, False]), "integer"),
    (torch.tensor([[0, 10]]), "(N+1,)"),
    (torch.tensor([10]), "(N+1,)"),
    ([0, 10], "integer tensor"),
])
def test_malformed_cu_seqlens_raise(cu, msg):
    H = _H()
    with pytest.raises(H.HyenaB200Error, match=msg.replace("[", r"\[").replace("(", r"\(").replace(")", r"\)")
                       .replace("+", r"\+")):
        _op()(torch.zeros(10, 8), cu_seqlens=cu)


def test_operator_validation_before_device_work():
    H = _H()
    op = _op()
    u = torch.zeros(10, 8)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    n0 = _lib.launch_count()
    for kw, msg in [(dict(lengths=[4, 6]), "lengths or mask"), (dict(mask=torch.ones(1, 10)), "lengths or mask"),
                    (dict(max_seqlen=5), "max_seqlen = 5 is shorter"),
                    (dict(inference_params=H.DecodeCache()), "DecodeCache")]:
        with pytest.raises(H.HyenaB200Error, match=msg):
            op(u, cu_seqlens=cu, **kw)
    with pytest.raises(H.HyenaB200Error, match="exceeds l_max"):
        H.HyenaOperator(8, 5, emb_dim=5)(u, cu_seqlens=cu)
    with pytest.raises(H.HyenaB200Error, match="order 2"):
        _op(order=3)(u, cu_seqlens=cu)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        _op(bidirectional=True)(u, cu_seqlens=cu)
    for bad in (torch.zeros(2, 5, 8), torch.zeros(10, 7), torch.zeros(1, 1, 10, 8)):
        with pytest.raises(H.HyenaB200Error, match="packed input"):
            op(bad, cu_seqlens=cu)
    with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):        # every check passes: the device is next
        op(u, cu_seqlens=cu, max_seqlen=6)
    assert _lib.launch_count() == n0


def test_block_and_backbone_validate_before_device_work():
    H = _H()
    mixer = partial(H.HyenaOperator, l_max=64, emb_dim=5)
    blk = H.Block(8, mixer_cls=mixer)
    bb = H.Backbone(8, 2, mixer)
    u = torch.zeros(10, 8)
    n0 = _lib.launch_count()
    with pytest.raises(H.HyenaB200Error, match="non-decreasing"):
        blk(u, mixer_kwargs={"cu_seqlens": torch.tensor([0, 6, 4, 10])})
    with pytest.raises(H.HyenaB200Error, match="max_seqlen"):
        blk(u, mixer_kwargs={"cu_seqlens": torch.tensor([0, 4, 10]), "max_seqlen": 2})
    with pytest.raises(H.HyenaB200Error, match="lengths or mask"):
        bb(u, mask=torch.ones(1, 10), cu_seqlens=torch.tensor([0, 10]))
    with pytest.raises(H.HyenaB200Error, match="cu_seqlens\\[0\\]"):
        bb(u, cu_seqlens=torch.tensor([2, 10]))
    with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
        bb(u, cu_seqlens=torch.tensor([0, 4, 10]))
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- truth self-check
def _leaky(u, dy, cu, P, kind):
    """Planted isolation bugs, fp64: "whole" convolves the whole packed row as one sequence; "short" lets the 3-tap filter
    read the previous sequence's last position (the operator on each sequence with that one position prepended)."""
    if kind == "whole":
        y, du, _ = O.operator_fwd_bwd(u[None].double(), O.to_dtype(P, torch.float64), dy[None].double())
        return {i: y[0, a:b] for i, (a, b) in enumerate(zip(cu[:-1], cu[1:]))}
    out = {}
    Q = O.to_dtype(P, torch.float64)
    for i, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        s = max(a - 1, 0)
        y, _, _ = O.operator_fwd_bwd(u[None, s:b].double(), Q, dy[None, s:b].double())
        out[i] = y[0, a - s:]
    return out


@pytest.mark.parametrize("kind", ["whole", "short"])
def test_per_sequence_truth_rejects_leaks(kind):
    D = 4
    g = torch.Generator().manual_seed(1)
    P = O.init_params(D, 64, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    P["in_proj.bias"] = 0.02 * torch.randn(P["in_proj.bias"].shape, generator=g)
    u, cu = packed_input([5, 9, 1, 17], D)
    dy = torch.randn(u.shape, generator=g)
    t32 = seq_truth(u, dy, cu, P, torch.float32)
    t64 = seq_truth(u, dy, cu, P, torch.float64)
    direct = {i: O.operator_fwd_bwd(u[None, a:b].double(), O.to_dtype(P, torch.float64), dy[None, a:b].double())[0][0]
              for i, (a, b) in enumerate(zip(cu[:-1], cu[1:]))}
    for i in t32[0]:                                    # the truth agrees with running each sequence alone
        PU.check(direct[i], t32[0][i], f"truth seq {i}", ref64=t64[0][i])
    bad = _leaky(u, dy, cu, P, kind)
    missed = 0
    for i in range(1, len(cu) - 1):
        try:
            PU.check(bad[i], t32[0][i], f"leak {kind} seq {i}", ref64=t64[0][i])
        except AssertionError:
            missed += 1
    PU._records[:] = [r for r in PU._records if not r["what"].startswith("leak")]
    assert missed == len(cu) - 2, f"the bar let a {kind} leak through"
