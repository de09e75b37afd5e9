"""Streaming forward on the GPU (``forward(u, stream=True)``, DESIGN.md section 4.21): every position of sequences past
l_max and past 2^20 positions, through HyenaOperator, Block and Backbone.

The truth is the operator's composition with its l_max-tap causal convolution over the whole sequence
(tests/test_stream_cpu.py:stream_truth), in fp64 through FFTs; the fp32 result is the same composition in fp32 (and, where
the sequence is short enough to decode, the unbounded DecodeCache's prefill + extends).  Every comparison goes through
tests/parity_util.py and is booked."""
from functools import partial

import pytest
import torch
import torch.nn.functional as F

from tests import parity_util as PU
from tests.test_stream_cpu import stream_truth

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _op(D, l_max, order=2, seed=0):
    torch.manual_seed(seed)
    op = _H().HyenaOperator(D, l_max, order=order, emb_dim=5, w=10.0)
    with torch.no_grad():
        op.in_proj.bias.normal_(0, 0.02)
    return op.to(_dev())


def _input(B, L, D, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.randn(B, L, D, generator=g, device=_dev())


def _ops():
    from hyena_dna_b200 import ops
    return ops


# ---------------------------------------------------------------------------------------------- the operator
CASES = [(o, lm, L, D) for o in (2, 3) for lm in (61, 1026, 4099, 1 << 16)
         for L, D in ((lm + 1, 100), (3 * lm + 5, 100), ((1 << 20) + 1, 3), ((1 << 21) + 3, 1))]
CASES += [(2, 1026, 1 << 20, 100), (3, 61, (1 << 20) + 1, 100), (2, 4099, (1 << 21) + 3, 3)]
# one window of L_b = 2^15 (LOGM1 = 5, the first two-level transform) for both orders, and of 2^19 for the plain passes
CASES += [(2, 4099, 20001, 100), (3, 4099, 20001, 100), (3, 1026, 300001, 3)]


@pytest.mark.parametrize("order,l_max,L,D", CASES)
def test_stream_operator(order, l_max, L, D):
    dev = _dev()
    op = _op(D, l_max, order, seed=l_max + L)
    B = 3
    u = _input(B, L, D, seed=L)
    with torch.no_grad():
        y = op(u, stream=True)
    assert y.shape == u.shape and y.dtype == u.dtype
    ref64 = stream_truth(op, u, torch.float64)
    ref32 = stream_truth(op, u, torch.float32)
    PU.check(y, ref32, f"stream o{order} l_max {l_max} L {L} D {D}", ref64=ref64)


@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("l_max", [61, 1026, 4099, 1 << 16])
def test_stream_dispatches_to_forward_up_to_l_max(order, l_max):
    op = _op(3, l_max, order, seed=7)
    for L in (l_max - 1, l_max):
        u = _input(3, L, 3, seed=L)
        with torch.no_grad():
            assert torch.equal(op(u, stream=True), op(u))


@pytest.mark.parametrize("order", [2, 3])
def test_rows_are_independent(order):
    """A NaN in one row changes no bit of the others."""
    op = _op(8, 1026, order, seed=3)
    u = _input(3, (1 << 20) + 1, 8, seed=5)
    with torch.no_grad():
        y = op(u, stream=True)
        u2 = u.clone()
        u2[1, 500000] = float("nan")
        y2 = op(u2, stream=True)
    assert torch.equal(y[0], y2[0]) and torch.equal(y[2], y2[2])
    assert torch.isnan(y2[1]).any()


@pytest.mark.parametrize("order,l_max", [(2, 61), (3, 61), (2, 1026), (3, 1026)])
def test_stream_agrees_with_an_unbounded_decode_cache(order, l_max):
    op = _op(16, l_max, order, seed=11)
    L = 3 * l_max + 5
    u = _input(3, L, 16, seed=13)
    with torch.no_grad():
        y = op(u, stream=True)
        c = op.allocate_decode_cache(3, None)
        P0 = l_max // 2
        yd = torch.cat([op.prefill(u[:, :P0], c), op.extend(u[:, P0:], c)], dim=1)
    PU.check(y, yd, f"stream vs decode o{order} l_max {l_max}", ref64=stream_truth(op, u, torch.float64))


@pytest.mark.parametrize("order,L_b", [(o, L_b) for o in (2, 3) for L_b in (2048, 8192, 1 << 15, 1 << 16, 1 << 19)])
def test_window_route_matches_one_window_of_the_whole_row(order, L_b):
    """Windows of L_b positions against the default plan of a row that fits, one window of 2^20: the same outputs up to
    rounding, and that window against the truth."""
    ops = _ops()
    op = _op(32, 1026, order, seed=17)
    L = (1 << 20) - 3
    u = _input(2, L, 32, seed=19)
    pl = ops.stream_plan(L, 1026, order, 2)
    assert pl.L_b == 1 << 20 and len(pl.chunks) == 1
    with torch.no_grad():
        y = op._forward_stream(u, ops.stream_plan(L, 1026, order, 2, L_b=L_b))
        y1 = op._forward_stream(u, pl)
    ref64 = stream_truth(op, u, torch.float64)
    PU.check(y, y1, f"o{order} windows of {L_b} vs one window", ref64=ref64)
    PU.check(y1, stream_truth(op, u, torch.float32), f"o{order} one window of 2^20", ref64=ref64)


def _chunked_plan(L, l_max, order, B, L_b, chunk_positions, short=0):
    """ops.stream_plan with small windows and chunks, so that several chunk edges fall inside the sequence; ``short``
    positions less chunk context than the plan's rule (the same chunk outputs, each chunk starting later)."""
    ops = _ops()
    pl = ops.stream_plan(L, l_max, order, B, L_b=L_b, chunk_positions=chunk_positions)
    assert len(pl.chunks) >= 3
    if not short:
        return pl
    cc = pl.chunk_context - short
    return ops.StreamPlan(pl.L, pl.l_max, pl.order, pl.B, pl.L_b, pl.context, cc,
                          [(max(0, a - cc), a, e) for _, a, e in pl.chunks])


@pytest.mark.parametrize("l_max,L,L_b,chunk_positions", [(61, 5000, 1024, 3000), (1026, 20001, 4096, 3 * 8192)])
def test_stream_order_4_across_chunk_edges(l_max, L, L_b, chunk_positions):
    """Order 4 (three windowed recurrences per chunk, chunk context 3 (l_max - 1) + 2) with chunks small enough that
    several chunk edges fall inside the sequence, against the truth."""
    op = _op(16, l_max, 4, seed=l_max)
    u = _input(3, L, 16, seed=L)
    with torch.no_grad():
        y = op._forward_stream(u, _chunked_plan(L, l_max, 4, 3, L_b, chunk_positions))
    PU.check(y, stream_truth(op, u, torch.float32), f"stream o4 l_max {l_max} L {L} chunked",
             ref64=stream_truth(op, u, torch.float64))


@pytest.mark.parametrize("order", [3, 4])
def test_truth_rejects_a_chunk_one_position_short_of_context(order):
    """The order >= 3 counterpart of test_stream_cpu.test_truth_rejects_a_plan_with_one_position_too_little_context: a
    StreamPlan whose chunks carry one position less than (order - 1)(l_max - 1) + 2 of context fails the bar the plan's
    own chunks pass.  The filter is random and does not decay, so its last tap, which the missing position reaches
    through, is not negligible."""
    l_max, L = 61, 5000
    op = _op(8, l_max, order, seed=order)
    k = torch.randn(8 * (order - 1), l_max, generator=torch.Generator(device=_dev()).manual_seed(5), device=_dev())
    op.filter_fn.filter_channel_major = lambda n: k[:, :n] / 4
    u = _input(2, L, 8, seed=order)
    ref64, ref32 = stream_truth(op, u, torch.float64), stream_truth(op, u, torch.float32)
    with torch.no_grad():
        good = op._forward_stream(u, _chunked_plan(L, l_max, order, 2, 1024, 2000))
        bad = op._forward_stream(u, _chunked_plan(L, l_max, order, 2, 1024, 2000, short=1))
    n0 = len(PU._records)
    try:
        PU.check(good, ref32, f"o{order} chunk context exact", ref64=ref64)
        with pytest.raises(AssertionError):
            PU.check(bad, ref32, f"o{order} chunk context one short", ref64=ref64)
    finally:
        del PU._records[n0:]            # a self-check of the bar, not a parity record


# ---------------------------------------------------------------------------------------------- Block and Backbone
def _ln(x, m):
    return F.layer_norm(x, (x.shape[-1],), m.weight.to(x.dtype), m.bias.to(x.dtype), m.eps)


def _mlp(x, m):
    h = F.gelu(F.linear(x, m.fc1.weight.to(x.dtype), m.fc1.bias.to(x.dtype)), approximate=m.approximate)
    return F.linear(h, m.fc2.weight.to(x.dtype), m.fc2.bias.to(x.dtype))


def _block_truth(blk, h, res, dt):
    res = h.to(dt) if res is None else h.to(dt) + res.to(dt)
    h = stream_truth(blk.mixer, _ln(res, blk.norm1), dt)
    res = h + res
    return _mlp(_ln(res, blk.norm2), blk.mlp), res


def _backbone(D, l_max, n_layer=2, seed=0):
    H = _H()
    torch.manual_seed(seed)
    m = H.Backbone(D, n_layer, partial(H.HyenaOperator, l_max=l_max, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True)
    return m.to(_dev())


def test_backbone_stream_past_2_20():
    bb = _backbone(32, 1026, 2, seed=23)
    u = _input(2, (1 << 20) + 5, 32, seed=29)
    with torch.no_grad():
        y = bb(u, stream=True)
    outs = {}
    for dt in (torch.float64, torch.float32):
        h, res = u, None
        for layer in bb.layers:
            h, res = _block_truth(layer, h, res, dt)
        outs[dt] = _ln(h + res, bb.ln_f)
    PU.check(y, outs[torch.float32], "backbone stream", ref64=outs[torch.float64])


def test_block_stream_through_mixer_kwargs():
    bb = _backbone(16, 4099, 1, seed=31)
    blk = bb.layers[0]
    u = _input(3, 3 * 4099 + 5, 16, seed=37)
    r = _input(3, 3 * 4099 + 5, 16, seed=41)
    with torch.no_grad():
        h, res = blk(u, r, mixer_kwargs={"stream": True})
        h0, res0 = blk(u[:, :4000], r[:, :4000], mixer_kwargs={"stream": True})
        hb, resb = blk(u[:, :4000], r[:, :4000])
    assert torch.equal(h0, hb) and torch.equal(res0, resb)
    h64, res64 = _block_truth(blk, u, r, torch.float64)
    h32, res32 = _block_truth(blk, u, r, torch.float32)
    PU.check(h, h32, "block stream h", ref64=h64)
    PU.check(res, res32, "block stream residual", ref64=res64)


# ---------------------------------------------------------------------------------------------- one large case
def test_large_stream_64bit_offsets():
    """B L D > 2^31: y at positions around window and chunk edges against an fp64 direct sum over each position's
    l_max + 1 positions of context."""
    ops = _ops()
    D, l_max, L = 256, 1026, (1 << 23) + 5
    op = _op(D, l_max, 2, seed=43)
    u = _input(1, L, D, seed=47)
    with torch.no_grad():
        y = op(u, stream=True)
    pl = ops.stream_plan(L, l_max, 2, 1)
    marks = set()
    for s, a, e in pl.chunks:
        marks.update((a, e - 1))
        for st, _, os_ in pl.windows(e - s)[:3] + pl.windows(e - s)[-3:]:
            marks.update((s + st + os_, s + st + pl.L_b - 1))
    ts = sorted({t + d for t in marks for d in (-2, -1, 0, 1, 2) if 0 <= t + d < L})
    got, r32, r64 = [], [], []
    for t in ts:
        s0 = max(0, t - l_max - 1)
        got.append(y[:, t])
        for dt, out in ((torch.float32, r32), (torch.float64, r64)):
            out.append(stream_truth(op, u[:, s0:t + 1], dt, positions=[t - s0])[:, 0])
    PU.check(torch.stack(got, 1), torch.stack(r32, 1), f"large stream at {len(ts)} positions",
             ref64=torch.stack(r64, 1))
