"""Continuous batching on the GPU (HyenaOperator.admit, Block.admit, Backbone.admit, DecodeCache.release / compact,
hyena_b200_decode_admit / _decode_shift; DESIGN.md section 4.15).  Admitted rows against prefill (bits) and the fp64
oracle on each request's unpadded tokens; the other rows against a twin cache (bits).  Tolerance policy:
tests/parity_util.py."""
from functools import partial

import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_ragged import _make, _padded

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _tokens(n, D, seed):
    return O.nucleotide_activations(1, n, D, seed=seed)[0][0]                 # (n, D) on the CPU


def _check_seq(ys, seq, P, n_new, what):
    """ys (n_new, D): outputs of the last n_new positions of the request seq (L, D) against the fp64 oracle."""
    r32 = O.hyena_operator(seq[None], P)[0, -n_new:]
    r64 = O.hyena_operator(seq[None].double(), O.to_dtype(P, torch.float64))[0, -n_new:]
    PU.check(ys.cpu(), r32, what, ref64=r64)


def _clone(c):
    """An independent copy of the operator cache c (same filter, copied state and host fields)."""
    n = type(c)(c.owner, c.batch_size, c.max_seqlen, c.lcap, c.k, c.bias, c.h.clone(), c.tail.clone(), c.s_t.clone(),
                c.part.clone())
    n.t, n.steps, n.win_b, n.win_wc = c.t, c.steps, c.win_b, c.win_wc
    n.win_f = None if c.win_f is None else c.win_f.clone()
    n.set_start(c.start)
    n._free = c._free
    return n


def _step_both(op, a, b, toks, rows_same):
    """Step caches a and b with the same tokens (B, n, D); the rows rows_same must give the same bits -> a's outputs."""
    out = []
    with torch.no_grad():
        for i in range(toks.shape[1]):
            ya, yb = op.step(toks[:, i:i + 1], a), op.step(toks[:, i:i + 1], b)
            assert torch.equal(ya[rows_same], yb[rows_same]), f"step {i}"
            out.append(ya)
    return torch.cat(out, 1)


# ---------------------------------------------------------------------------------------------- 1. admission
ADMIT = [(2, 8, 1), (2, 8, 9), (2, 100, 5), (2, 256, 17), (3, 8, 2), (3, 100, 8), (3, 256, 16), (2, 100, 16)]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("order,D,B", ADMIT)
def test_admit_bits_state_and_decoding(order, D, B, ragged):
    dev = _dev()
    H = _H()
    op, P = _make(D, 4096, order)
    t0, Pn = 1200, 700
    k = min(B, 3)
    rows = list(range(B - 1, B - 1 - k, -1))                            # the last rows, in reverse order
    lens0 = [t0 - 37 * b % t0 for b in range(B)]
    u0 = _padded(B, t0, D, lens0, seed=1).to(dev)
    a, b = op.allocate_decode_cache(B, 4096), op.allocate_decode_cache(B, 4096)
    with torch.no_grad():
        op.prefill(u0, a, lengths=lens0)
        op.prefill(u0, b, lengths=lens0)
    lens = [Pn - 113 * i for i in range(k)] if ragged else None
    u = _padded(k, Pn, D, lens or [Pn] * k, seed=2).to(dev)
    fresh = op.allocate_decode_cache(k, Pn)
    with torch.no_grad():
        y_ref = op.prefill(u, fresh, lengths=lens)
        y = op.admit(u, a, rows, lengths=lens)
    assert torch.equal(y, y_ref)
    off, others = t0 - Pn, [r for r in range(B) if r not in rows]
    for i, r in enumerate(rows):
        assert not a.h[:, r, :, :off].any()
        assert torch.equal(a.h[:, r, :, off:t0], fresh.h[:, i, :, :Pn]), f"h of row {r}"
        assert torch.equal(a.tail[r], fresh.tail[i]), f"tail of row {r}"
    assert torch.equal(a.h[:, others], b.h[:, others]) and torch.equal(a.tail[others], b.tail[others])
    n_lens = lens or [Pn] * k
    assert a.t == t0 and a.lengths == tuple(n_lens[rows.index(r)] if r in rows else lens0[r] for r in range(B))
    # steps, then a direct and an FFT extend: the other rows give the twin's bits, the admitted rows the oracle's values
    toks = torch.stack([_tokens(3 + 5 + 600, D, seed=10 + r) for r in range(B)]).to(dev)
    ys = [_step_both(op, a, b, toks[:, :3], others)]
    for lo, hi in ((3, 8), (8, 608)):
        with torch.no_grad():
            ya, yb = op.extend(toks[:, lo:hi], a), op.extend(toks[:, lo:hi], b)
        assert torch.equal(ya[others], yb[others])
        ys.append(ya)
    ys = torch.cat(ys, 1)
    for i, r in enumerate(rows):
        seq = torch.cat([u[i, Pn - n_lens[i]:].cpu(), toks[r].cpu()])
        _check_seq(ys[r], seq, P, toks.shape[1], f"order {order} D {D} B {B} row {r}")


# ---------------------------------------------------------------------------------------------- 2. shifts
@pytest.mark.parametrize("lcap", [1000, 1001, 1002, 1003])
def test_decode_shift_matches_slices(lcap):
    dev = _dev()
    H = _H()
    op, _ = _make(8, 2048, 3)
    c = op.allocate_decode_cache(5, lcap)
    g = torch.Generator(device=dev).manual_seed(lcap)
    for t, shift in ((lcap, -4), (lcap, -(lcap - lcap % 4)), (777, -400), (777, -776), (777, 4), (600, 400),
                     (5, 4 * ((lcap - 8) // 4)), (1, 8), (333, -332)):
        if t + shift > lcap or shift < -t:
            continue
        c.h.copy_(torch.randn(c.h.shape, generator=g, device=dev))
        before = c.h.clone()
        c.t, T4 = t, (t + 3) // 4 * 4
        c.set_start(None)
        H.ops.decode_shift(c, shift)
        want = before.clone()
        if shift < 0:
            want[..., :T4 + shift] = before[..., -shift:T4]
        else:
            want[..., shift:T4 + shift] = before[..., :T4]
            want[..., :shift] = 0.0
        assert torch.equal(c.h, want), (lcap, t, shift)
        assert c.t == t + shift


def _long_cache(op, B, t0, D, seed):
    """A B-row cache of op prefilled with t0 random positions, stepped until a window holds the position."""
    dev = _dev()
    H = _H()
    u = O.nucleotide_activations(B, t0, D, seed=seed)[0].to(dev)
    c = op.allocate_decode_cache(B, 1 << 17)
    with torch.no_grad():
        op.prefill(u, c)
        for i in range(H.ops.WINDOW_AFTER_STEPS + 24):
            op.step(_tokens(B, D, seed + 1 + i)[:, None].to(dev), c)
    assert c.win_wc > 0 and c.win_b <= c.t
    return c, u


def test_window_admission_and_compaction():
    dev = _dev()
    H = _H()
    D, B, t0 = 8, 3, (1 << 16) + 40
    op, P = _make(D, 1 << 17, 2)
    a, u0 = _long_cache(op, B, t0, D, seed=5)
    b = _clone(a)
    t = a.t
    # prompt 1 starts after the window base (its F is zero), prompt 2 before it (F from its history)
    p1, p2 = _tokens(8, D, 71), _tokens(3000, D, 72)
    assert t - 8 >= a.win_b > t - 3000
    with torch.no_grad():
        op.admit(p1[None].to(dev), a, [0])
        op.admit(p2[None].to(dev), a, [2])
    assert a.win_wc == b.win_wc and a.win_b == b.win_b and a.t == t
    assert torch.equal(a.win_f[:, 1], b.win_f[:, 1]) and not a.win_f[:, 0, :, :a.win_wc].any()
    toks = torch.stack([_tokens(20, D, 80 + r) for r in range(B)]).to(dev)
    ys = _step_both(op, a, b, toks, [1])
    _check_seq(ys[0], torch.cat([p1, toks[0].cpu()]), P, 20, "window: prompt after win_b")
    _check_seq(ys[2], torch.cat([p2, toks[2].cpu()]), P, 20, "window: prompt before win_b")
    # compaction that keeps the window: the same bits as the uncompacted twin on every row
    a.release([1])
    twin = _clone(a)
    m = a.compact()
    assert m == (a.t + m - 3000 - 20) // 4 * 4 and m > 0 and a.win_wc == twin.win_wc and a.win_b == twin.win_b - m
    more = torch.stack([_tokens(12, D, 90 + r) for r in range(B)]).to(dev)
    ys2 = _step_both(op, a, twin, more, [0, 1, 2])
    _check_seq(ys2[2], torch.cat([p2, toks[2].cpu(), more[2].cpu()]), P, 12, "window kept through compaction")
    # releasing the long row makes m > win_b: the window closes and the steps go on the plain route, still right
    a.release([2])
    m2 = a.compact()
    assert m2 > 0 and (a.win_b, a.win_wc) == (0, 0) and a.lengths[0] == 8 + 20 + 12
    last = _tokens(6, D, 99)
    with torch.no_grad():
        y = torch.cat([op.step(last[i][None, None].expand(B, 1, D).contiguous().to(dev), a) for i in range(6)], 1)
    _check_seq(y[0], torch.cat([p1, toks[0].cpu(), more[0].cpu(), last]), P, 6, "after the window closed")


def test_compaction_on_the_plain_route_and_right_shifts():
    dev = _dev()
    H = _H()
    D, B = 16, 4
    op, P = _make(D, 4096, 3)
    c = op.allocate_decode_cache(B, 4096)
    # a fresh cache: the clock moves to P, the rows that took no prompt are free
    pr = [_tokens(50, D, 200 + i) for i in range(2)]
    with torch.no_grad():
        op.admit(torch.stack(pr).to(dev), c, [0, 2])
    assert c.t == 50 and c.free == frozenset({1, 3}) and c.lengths == (50, 0, 50, 0)
    reqs = {0: [pr[0]], 2: [pr[1]]}
    # a longer prompt shifts every row right by 300 - 50 = 250 rounded up to 252
    p3 = _tokens(300, D, 210)
    with torch.no_grad():
        op.admit(p3[None].to(dev), c, [1])
    assert c.t == 302 and c.start[0] == 252 and c.start[1] == 2
    reqs[1] = [p3]
    outs = {r: [] for r in reqs}

    def run(n, seed):
        toks = torch.stack([_tokens(n, D, seed + r) for r in range(B)])
        with torch.no_grad():
            for i in range(n):
                y = op.step(toks[:, i:i + 1].to(dev), c)
                for r in reqs:
                    outs[r].append(y[r, 0].cpu())
        for r in reqs:
            reqs[r].append(toks[r])
    run(10, 300)
    c.release([1])
    reqs.pop(1), outs.pop(1)
    assert c.compact() == 252 and c.t == 60
    run(10, 400)
    for r in reqs:
        seq = torch.cat(reqs[r])
        _check_seq(torch.stack(outs[r]), seq, P, 20, f"row {r} through a right shift and a compaction")


# ---------------------------------------------------------------------------------------------- 3. sustained serving
def test_sustained_serving_past_lcap():
    dev = _dev()
    H = _H()
    D, B, lcap = 8, 4, 8192
    op, P = _make(D, lcap, 2)
    c = op.allocate_decode_cache(B, lcap)
    rng = torch.Generator().manual_seed(7)
    bank = _tokens(20000, D, 50000)
    live, done, advance, nreq = {}, 0, 0, 0

    def admit(r):
        nonlocal nreq
        n = int(torch.randint(100, 2000, (1,), generator=rng))
        gen = int(torch.randint(50, 400, (1,), generator=rng))
        p = _tokens(n, D, 1000 + nreq)
        nreq += 1
        if c.t + gen > lcap or n > max(c.t, 1) and c.t + (n - c.t + 3) // 4 * 4 > lcap:
            c.compact()
        with torch.no_grad():
            op.admit(p[None].to(dev), c, [r])
        live[r] = dict(seq=[p], ys=[], left=gen)
    for r in range(B):
        admit(r)
    while advance < 2 * lcap + 1000 or live:
        if c.t >= lcap - 1:
            assert c.compact() > 0
        tok = bank[(advance * B + torch.arange(B)) % bank.shape[0]]
        with torch.no_grad():
            y = op.step(tok[:, None].to(dev), c)
        advance += 1
        for r in list(live):
            q = live[r]
            q["seq"].append(tok[r:r + 1])
            q["ys"].append(y[r, 0].cpu())
            q["left"] -= 1
            if q["left"] == 0:
                seq = torch.cat(q["seq"])
                n = len(q["ys"])
                _check_seq(torch.stack(q["ys"]), seq, P, n, f"request in row {r} ({seq.shape[0]} positions)")
                done += 1
                del live[r]
                c.release([r])
                if advance < 2 * lcap:
                    admit(r)
    assert advance > 2 * lcap and done >= 2 * B


# ---------------------------------------------------------------------------------------------- 4. graphs and isolation
def test_step_graph_admits_releases_and_compacts_without_recapture():
    dev = _dev()
    H = _H()
    D, B, lcap = 32, 3, 4096
    torch.manual_seed(0)
    bb = H.Backbone(D, 2, partial(H.HyenaOperator, l_max=lcap, emb_dim=5, w=10.0),
                    mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
    ce, cg = bb.allocate_decode_cache(B, lcap), bb.allocate_decode_cache(B, lcap)
    u = O.nucleotide_activations(B, 400, D, seed=3)[0].to(dev)
    lens = [400, 120, 250]
    with torch.no_grad():
        for c in (ce, cg):
            bb.prefill(u, c, lengths=lens)
    graph = H.StepGraph(bb, cg)
    graphs, keys = dict(graph._graphs), dict(graph._keys)
    x = O.nucleotide_activations(B, 200, D, seed=4)[0].to(dev)

    def steps(lo, hi):
        with torch.no_grad():
            for i in range(lo, hi):
                ye = bb.step(x[:, i:i + 1], ce)
                yg = graph.step(x[:, i:i + 1])
                assert torch.equal(ye, yg), f"step {i}"
    steps(0, 20)
    p = O.nucleotide_activations(1, 300, D, seed=9)[0].to(dev)
    with torch.no_grad():
        ya, yb = bb.admit(p, ce, [1]), bb.admit(p, cg, [1])
    assert torch.equal(ya, yb)
    fresh = bb.allocate_decode_cache(1, 300)
    with torch.no_grad():
        assert torch.equal(ya, bb.prefill(p, fresh))
    steps(20, 60)
    for c in (ce, cg):
        c.release([0])
        assert c.compact() == 120                      # the live rows start at 120 (row 1) and 150 (row 2)
    steps(60, 100)
    with torch.no_grad():
        for c in (ce, cg):
            bb.admit(x[:1, :100], c, [0])
    steps(100, 140)
    assert graph._graphs == graphs and graph._keys == keys
    for a, b in zip(ce.layers, cg.layers):
        assert a.t == b.t and torch.equal(a.h, b.h) and torch.equal(a.tail, b.tail)


@pytest.mark.parametrize("fill", ["nan", "inf"])
def test_non_finite_prompt_stays_in_its_row(fill):
    dev = _dev()
    D, B = 16, 4
    op, _ = _make(D, 2048, 2)
    u0 = O.nucleotide_activations(B, 500, D, seed=1)[0].to(dev)
    a, b = op.allocate_decode_cache(B, 2048), op.allocate_decode_cache(B, 2048)
    with torch.no_grad():
        op.prefill(u0, a)
        op.prefill(u0, b)
    p = _tokens(200, D, 5)
    bad = p.clone()
    bad[50:60] = float("nan") if fill == "nan" else float("inf")
    with torch.no_grad():
        op.admit(bad[None].to(dev), a, [2])
        op.admit(p[None].to(dev), b, [2])
    others = [0, 1, 3]
    assert torch.equal(a.h[:, others], b.h[:, others]) and torch.equal(a.tail[others], b.tail[others])
    toks = torch.stack([_tokens(8, D, 40 + r) for r in range(B)]).to(dev)
    ys = _step_both(op, a, b, toks, others)
    assert torch.isfinite(ys[others]).all()


def test_profiler_counts_one_launch_per_layer():
    dev = _dev()
    H = _H()
    D, B, n_layer = 16, 2, 3
    torch.manual_seed(0)
    bb = H.Backbone(D, n_layer, partial(H.HyenaOperator, l_max=2048, emb_dim=5, w=10.0)).to(dev)
    c = bb.allocate_decode_cache(B, 2048)
    with torch.no_grad():
        bb.prefill(O.nucleotide_activations(B, 300, D, seed=1)[0].to(dev), c)
        p = O.nucleotide_activations(1, 100, D, seed=2)[0].to(dev)
        H._lib.profile_begin()
        bb.admit(p, c, [1])
        prof = H._lib.profile_end()
    assert prof["decode_hist"][1] == n_layer
    c.release([0])
    torch.cuda.synchronize()
    n0 = H.launch_count()
    assert c.compact() == 200
    assert H.launch_count() - n0 == n_layer
