"""Packed prompts into a decode cache on the GPU (``prefill`` / ``admit`` with ``cu_seqlens=`` of HyenaOperator, Block and
Backbone; hyena_b200_decode_admit_packed; DESIGN.md section 4.19).  Outputs against ``forward(u, cu_seqlens=...)`` (bits),
the cache against the left-padded route's (bits), decoding after it against the left-padded cache (bits) and against the
fp64 oracle on each whole sequence on the device, with the fp32 oracle as ``ref32`` (tests/test_decode_packed_cpu
.decode_truth).  Tolerance policy: tests/parity_util.py."""
from functools import partial

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_decode_packed_cpu import decode_truth
from tests.test_gpu_block_paths import _leaves, _ln_randomize
from tests.test_gpu_decode_admit import _clone
from tests.test_gpu_decode_paths import backbone_ref
from tests.test_gpu_ragged import _make
from tests.test_gpu_widths import _act
from tests.test_varlen_cpu import packed_input

pytestmark = pytest.mark.gpu

HIST = [torch.float32, torch.float16, torch.bfloat16]


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _cu(lengths):
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    return cu


def _pad_left(u, cu, P):
    """The packed prompts (total, D) left-padded to P -> (N, P, D), random pads."""
    g = torch.Generator(device=u.device).manual_seed(17)
    out = 3.0 * torch.randn(len(cu) - 1, P, u.shape[-1], generator=g, device=u.device)
    for i, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        out[i, P - (b - a):] = u[a:b]
    return out


def _same_state(a, b, what, rows=None):
    """Two operator caches hold the same bits (all rows, or ``rows``) and the same host fields."""
    r = slice(None) if rows is None else rows
    assert torch.equal(a.h[:, r], b.h[:, r]), f"{what}: h"
    assert torch.equal(a.tail[r], b.tail[r]), f"{what}: tail"
    assert a.t == b.t and (a.win_b, a.win_wc) == (b.win_b, b.win_wc), f"{what}: position or window"
    if rows is None:
        assert a.start == b.start and a.free == b.free, f"{what}: starts {a.start} vs {b.start}"
    if a.win_f is not None and a.win_wc:
        assert torch.equal(a.win_f[:, r, :, :a.win_wc], b.win_f[:, r, :, :b.win_wc]), f"{what}: win_f"


def _steps(op, caches, toks):
    """The same tokens (N, n, D) stepped on every cache: the same bits on each -> the outputs."""
    out = []
    with torch.no_grad():
        for i in range(toks.shape[1]):
            ys = [op.step(toks[:, i:i + 1], c) for c in caches]
            for y in ys[1:]:
                assert torch.equal(y, ys[0]), f"step {i}"
            out.append(ys[0])
    return torch.cat(out, 1)


def _schedule(op, caches, toks):
    """Steps, a direct and an FFT extend, then steps: bits equal on every cache -> outputs (N, n, D)."""
    H = _H()
    nf = H.ops.EXTEND_FFT_MIN_N
    cut = [0, 3, 8, 8 + nf, 8 + nf + 3]
    assert not H.ops.decode_extend_uses_fft(1, 5) and H.ops.decode_extend_uses_fft(1, nf)
    ys = [_steps(op, caches, toks[:, :3])]
    for lo, hi in ((3, 8), (8, 8 + nf)):
        with torch.no_grad():
            ye = [op.extend(toks[:, lo:hi], c) for c in caches]
        for y in ye[1:]:
            assert torch.equal(y, ye[0]), f"extend [{lo}, {hi})"
        ys.append(ye[0])
    ys.append(_steps(op, caches, toks[:, cut[3]:cut[4]]))
    return torch.cat(ys, 1)


def _check_decoding(ys, u, cu, toks, P, what, only=None):
    dev = _dev()
    prompts = [u[a:b] for a, b in zip(cu[:-1], cu[1:])]
    conts = list(toks)
    sel = range(len(prompts)) if only is None else only
    t32 = decode_truth([prompts[i] for i in sel], [conts[i] for i in sel], P, torch.float32, dev)
    t64 = decode_truth([prompts[i] for i in sel], [conts[i] for i in sel], P, torch.float64, dev)
    for j, i in enumerate(sel):
        PU.check(ys[i], t32[j], f"{what} seq {i} (prompt {cu[i + 1] - cu[i]})", ref64=t64[j])


# ---------------------------------------------------------------------------------------------- 1. operator prefill
def _edges(hi):
    out, k = [1, 2, 3], 1024
    while k <= hi:
        out += [k - 1, k, k + 1] if k < hi else [k - 1, k]
        k *= 2
    return out


CASES = {
    "edges_2e17": (8, 1 << 18, _edges(1 << 17)),
    "starts_mod4_d1": (1, 8192, [3, 1, 2, 5, 1026, 7, 1023, 2049, 2, 1, 4096]),
    "starts_mod4_d5": (5, 8192, [3, 1, 2, 5, 1026, 7, 1023, 2049, 2, 1, 4096]),
    "d256": (256, 8192, [1, 2, 3, 1023, 1024, 1025, 4095, 6]),
}


@pytest.mark.parametrize("hist", HIST, ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("case", list(CASES))
def test_operator_prefill_bits_cache_and_decoding(case, hist):
    dev = _dev()
    D, lcap, lengths = CASES[case]
    op, Pp = _make(D, lcap)
    u, cu = packed_input(lengths, D)
    u = u.to(dev)
    cut = torch.tensor(cu, dtype=torch.int32)
    N, P = len(lengths), max(lengths)
    a, b = op.allocate_decode_cache(N, lcap, hist), op.allocate_decode_cache(N, lcap, hist)
    with torch.no_grad():
        y = op.prefill(u, a, cu_seqlens=cut)
        y_fwd = op(u, cu_seqlens=cut)
        op.prefill(_pad_left(u, cu, P), b, lengths=lengths)
    assert torch.equal(y, y_fwd), "prefill output differs from forward(u, cu_seqlens)"
    _same_state(a, b, "packed vs left-padded prefill")
    assert a.t == P and a.start == tuple(P - n for n in lengths) and a.win_wc == 0
    toks = O.nucleotide_activations(N, 16 + _H().ops.EXTEND_FFT_MIN_N, D, seed=31)[0].to(dev)
    ys = _schedule(op, [a, b], toks)
    if hist == torch.float32:
        _check_decoding(ys, u, cu, toks[:, :ys.shape[1]], Pp, f"{case} decode")


def test_prefill_of_a_2e20_prompt():
    dev = _dev()
    D, lcap = 8, 1 << 20
    op, Pp = _make(D, lcap)
    lengths = [3, lcap, 1025]
    u, cu = packed_input(lengths, D)
    u = u.to(dev)
    a, b = op.allocate_decode_cache(3, lcap), op.allocate_decode_cache(3, lcap)
    with torch.no_grad():
        y = op.prefill(u, a, cu_seqlens=torch.tensor(cu), max_seqlen=lcap)
        assert torch.equal(y, op(u, cu_seqlens=torch.tensor(cu)))
        op.prefill(_pad_left(u, cu, lcap), b, lengths=lengths)
    _same_state(a, b, "2^20 prefill")
    c = op.allocate_decode_cache(3, lcap)
    lengths2 = [3, lcap - 8, 1025]
    u2, cu2 = packed_input(lengths2, D, seed=1)
    u2 = u2.to(dev)
    with torch.no_grad():
        op.prefill(u2, c, cu_seqlens=torch.tensor(cu2))
    toks = O.nucleotide_activations(3, 6, D, seed=32)[0].to(dev)
    ys = _steps(op, [c], toks)
    _check_decoding(ys, u2, cu2, toks, Pp, "2^20 - 8 prompt then steps", only=[0, 2])


# ---------------------------------------------------------------------------------------------- 2. 64-bit offsets
def test_prefill_64bit_offsets():
    dev = _dev()
    D, lcap = 256, 1 << 20
    lengths = [1 << 20, 1 << 20, 700000, 1000]
    assert 3 * D * sum(lengths) > 2 ** 31
    op, Pp = _make(D, lcap)
    u, cu = packed_input(lengths, D)
    u = u.to(dev)
    a = op.allocate_decode_cache(4, lcap)
    with torch.no_grad():
        y = op.prefill(u, a, cu_seqlens=torch.tensor(cu, dtype=torch.int64, device=dev))
        assert torch.equal(y, op(u, cu_seqlens=torch.tensor(cu)))
    with torch.no_grad():
        b = op.allocate_decode_cache(4, lcap)
        op.prefill(_pad_left(u, cu, lcap), b, lengths=lengths)
        _same_state(a, b, "64-bit offsets")
        del b
        torch.cuda.empty_cache()
    a.release([0, 1])                                  # the cache is full: make room behind the two short prompts
    assert a.compact() == (lcap - 700000) // 4 * 4
    toks = O.nucleotide_activations(4, 4, D, seed=33)[0].to(dev)
    ys = _steps(op, [a], toks)
    _check_decoding(ys, u, cu, toks, Pp, "64-bit offsets decode", only=[3])


# ---------------------------------------------------------------------------------------------- 3. windows and graphs
def test_windowed_steps_and_step_graph_after_packed_prefill():
    dev = _dev()
    H = _H()
    D, lcap = 8, 1 << 17
    op, Pp = _make(D, lcap)
    lengths = [(1 << 16) + 40, 5, 30000]
    u, cu = packed_input(lengths, D)
    u = u.to(dev)
    a, g, b, bg = (op.allocate_decode_cache(3, lcap) for _ in range(4))
    with torch.no_grad():
        for c in (a, g):
            op.prefill(u, c, cu_seqlens=torch.tensor(cu))
        for c in (b, bg):
            op.prefill(_pad_left(u, cu, max(lengths)), c, lengths=lengths)
    # a graph opens the window at once, eager steps after WINDOW_AFTER_STEPS: compare each route with itself
    graph, graph_b = H.StepGraph(op, g), H.StepGraph(op, bg)
    n = H.ops.WINDOW_AFTER_STEPS + 24
    toks = O.nucleotide_activations(3, n, D, seed=34)[0].to(dev)
    out, outg = [], []
    with torch.no_grad():
        for i in range(n):
            ya, yb = op.step(toks[:, i:i + 1], a), op.step(toks[:, i:i + 1], b)
            yg = graph.step(toks[:, i:i + 1]).clone()
            ygb = graph_b.step(toks[:, i:i + 1])
            assert torch.equal(ya, yb) and torch.equal(yg, ygb), f"step {i}"
            out.append(ya)
            outg.append(yg)
    assert a.win_wc > 0 and g.win_wc > 0 and a.t >= 1 << 16
    _check_decoding(torch.cat(out, 1), u, cu, toks, Pp, "windowed steps")
    _check_decoding(torch.cat(outg, 1), u, cu, toks, Pp, "StepGraph steps")


# ---------------------------------------------------------------------------------------------- 4. admission
def _running(op, B, t0, D, lcap, window):
    """A B-row cache at position t0 (prefilled with left-padded prompts), with a window open or not."""
    H = _H()
    dev = _dev()
    lens0 = [t0 - 37 * r % max(t0 // 2, 1) for r in range(B)]
    u0 = O.nucleotide_activations(B, t0, D, seed=40)[0].to(dev)
    c = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(u0, c, lengths=lens0)
        if window:
            for i in range(H.ops.WINDOW_AFTER_STEPS + 4):
                op.step(O.nucleotide_activations(B, 1, D, seed=41 + i)[0].to(dev), c)
    assert (c.win_wc > 0) == window
    return c


@pytest.mark.parametrize("window", [False, True], ids=["closed", "open"])
@pytest.mark.parametrize("where", ["p_lt_t", "p_gt_t", "t0"])
def test_admission_matches_left_padded_admit(where, window):
    if where == "t0" and window:
        pytest.skip("a fresh cache has no window")
    dev = _dev()
    H = _H()
    D, B, lcap = 16, 5, 1 << 17
    op, Pp = _make(D, lcap)
    t0 = {"p_lt_t": 9000, "p_gt_t": 2000, "t0": 0}[where] + ((1 << 16) if window else 0)  # a window opens at long t only
    lengths = [700, 1, t0 + 1001 if where == "p_gt_t" else 3001, 2]
    rows = [4, 0, 2, 1]
    if t0:
        a = _running(op, B, t0, D, lcap, window)
    else:
        a = op.allocate_decode_cache(B, lcap)
    b, before = _clone(a), _clone(a)
    u, cu = packed_input(lengths, D, seed=3)
    u = u.to(dev)
    P = max(lengths)
    with torch.no_grad():
        y = op.admit(u, a, rows, cu_seqlens=torch.tensor(cu))
        op.admit(_pad_left(u, cu, P), b, rows, lengths=lengths)
        assert torch.equal(y, op(u, cu_seqlens=torch.tensor(cu)))
    _same_state(a, b, f"admission {where} window {window}")
    others = [r for r in range(B) if r not in rows]
    shift = a.t - before.t if t0 else 0
    for r in others:
        assert torch.equal(a.tail[r], before.tail[r]), f"tail of row {r}"
        assert torch.equal(a.h[:, r, :, shift:shift + before.t], before.h[:, r, :, :before.t]), f"h of row {r}"
        if window and a.win_wc:
            assert torch.equal(a.win_f[:, r, :, :a.win_wc], before.win_f[:, r, :, :a.win_wc]), f"win_f of row {r}"
    toks = O.nucleotide_activations(B, 24, D, seed=42)[0].to(dev)
    ys = _steps(op, [a, b], toks)
    _check_decoding(ys[rows], u, cu, toks[rows], Pp, f"admitted {where} window {window}")


def test_step_graph_captured_before_packed_admission_replays():
    dev = _dev()
    H = _H()
    D, B, lcap = 16, 4, 1 << 14
    op, _ = _make(D, lcap)
    ce = _running(op, B, 3000, D, lcap, False)
    cg = _clone(ce)
    graph = H.StepGraph(op, cg)
    x = O.nucleotide_activations(B, 60, D, seed=50)[0].to(dev)

    def steps(lo, hi):
        with torch.no_grad():
            for i in range(lo, hi):
                assert torch.equal(op.step(x[:, i:i + 1], ce), graph.step(x[:, i:i + 1])), f"step {i}"
    steps(0, 10)
    graphs, keys = dict(graph._graphs), dict(graph._keys)
    u, cu = packed_input([500, 3], D, seed=4)
    with torch.no_grad():
        for c in (ce, cg):
            op.admit(u.to(dev), c, [3, 1], cu_seqlens=torch.tensor(cu))
    steps(10, 40)
    ce.release([0])
    cg.release([0])
    steps(40, 60)
    assert graph._graphs == graphs and graph._keys == keys
    _same_state(ce, cg, "graph vs eager after a packed admission")


# ---------------------------------------------------------------------------------------------- 5. isolation
@pytest.mark.parametrize("fill", ["nan", "inf"])
def test_non_finite_prompt_stays_in_its_row(fill):
    dev = _dev()
    D = 16
    op, _ = _make(D, 4096)
    lengths = [300, 1030, 7, 2049]
    u, cu = packed_input(lengths, D)
    bad = u.clone()
    if fill == "nan":
        bad[cu[1]:cu[2]:2] = float("nan")
    else:
        g = torch.Generator().manual_seed(1)
        bad[cu[1]:cu[2]] = torch.where(torch.rand(lengths[1], D, generator=g) < 0.5, float("inf"), float("-inf"))
    a, b = op.allocate_decode_cache(4, 4096), op.allocate_decode_cache(4, 4096)
    with torch.no_grad():
        op.prefill(bad.to(dev), a, cu_seqlens=torch.tensor(cu))
        op.prefill(u.to(dev), b, cu_seqlens=torch.tensor(cu))
    _same_state(a, b, f"{fill} prompt", rows=[0, 2, 3])
    toks = O.nucleotide_activations(4, 8, D, seed=5)[0].to(dev)
    ya, yb = _steps(op, [a], toks), _steps(op, [b], toks)
    assert torch.equal(ya[[0, 2, 3]], yb[[0, 2, 3]]) and torch.isfinite(ya[[0, 2, 3]]).all()


# ---------------------------------------------------------------------------------------------- 6. Block and Backbone
def _backbone(D, l_max, seed=3):
    H = _H()
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mixer = partial(H.HyenaOperator, l_max=l_max, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh"))
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    _ln_randomize(m, g)
    return m.to(_dev())


def _backbone_truth(m, x, cu, what, y):
    """y against the fp64 composition on each sequence alone.  At D = 3 (LayerNorm over three features) the packed
    forward itself -- y has the bits of Backbone.forward(x, cu_seqlens) -- misses the elementwise bound against fp64 on a
    few elements in 10^4 more often than the fp32 composition does, and its largest error reaches 2.6x the fp32
    composition's (DESIGN.md section 4.19, an open finding about the packed forward at this width); there the check is
    that error within 4x, normwise within 2e-5."""
    dev = _dev()
    out = {}
    for bits, dt in ((32, torch.float32), (64, torch.float64)):
        sd = _leaves(m, dev, dt)
        out[bits] = torch.cat([backbone_ref(x[a:b][None].to(dev, dt), sd, 2, dt)[0] for a, b in zip(cu[:-1], cu[1:])])
    if x.shape[-1] > 3:
        _act(y, out[32], out[64], what)
        return
    e_ours = float((y.double() - out[64]).abs().max())
    e_ref = float((out[32].double() - out[64]).abs().max())
    nrm = float((y.double() - out[64]).norm() / out[64].norm())
    assert bool(torch.isfinite(y).all()) and e_ours <= 4 * e_ref and nrm <= 2e-5, (what, e_ours, e_ref, nrm)


@pytest.mark.parametrize("D", [3, 100])
def test_backbone_packed_prefill_and_admit(D):
    """The first layer's cache is the left-padded prefill's bit for bit (it depends on the in_proj products only); a later
    layer's input is the earlier layers' output, whose bits follow each prompt's transform size (its own bucket when
    packed, the longest prompt's when left-padded), so its cache is bit-identical only when the two sizes agree: all
    prompts in the bucket of P = 4096."""
    dev = _dev()
    H = _H()
    lcap = 8192
    m = _backbone(D, lcap)
    for lengths, same_all in (([700, 1, 1025, 3, 4096, 33], False), ([4096, 2049, 3000, 2500, 4001, 2050], True)):
        cu = _cu(lengths)
        x = torch.randn(cu[-1], D, generator=torch.Generator().manual_seed(7)).to(dev)
        cut = torch.tensor(cu, dtype=torch.int32, device=dev)
        a, b = m.allocate_decode_cache(6, lcap), m.allocate_decode_cache(6, lcap)
        with torch.no_grad():
            y = m.prefill(x, a, cu_seqlens=cut, max_seqlen=4096)
            assert torch.equal(y, m(x, cu_seqlens=cut))
            m.prefill(_pad_left(x, cu, max(lengths)), b, lengths=lengths)
        for la, lb in list(zip(a.layers, b.layers))[:None if same_all else 1]:
            _same_state(la, lb, f"backbone D {D} layer cache ({'one bucket' if same_all else 'mixed'})")
        _backbone_truth(m, x, cu, f"backbone D {D} packed prefill", y)
    # through Block, layer by layer, into a third cache: the same bits as the Backbone's
    c = m.allocate_decode_cache(6, lcap)
    with torch.no_grad():
        h, res = x, None
        for layer, lc in zip(m.layers, c.layers):
            h, res = layer.prefill(h, res, lc, cu_seqlens=cut, max_seqlen=4096)
        yc, _ = H.Block._add_norm(h, res, m.ln_f)
    assert torch.equal(yc, y)
    for la, lc in zip(a.layers, c.layers):
        _same_state(la, lc, f"block D {D} layer cache")
    # admission of two packed prompts into rows 5 and 1 of both caches
    lens2 = [50, 1004]
    cu2 = _cu(lens2)
    x2 = torch.randn(cu2[-1], D, generator=torch.Generator().manual_seed(5)).to(dev)
    with torch.no_grad():
        y2 = m.admit(x2, a, [5, 1], cu_seqlens=torch.tensor(cu2))
        m.admit(_pad_left(x2, cu2, max(lens2)), b, [5, 1], lengths=lens2)
        assert torch.equal(y2, m(x2, cu_seqlens=torch.tensor(cu2)))
    _same_state(a.layers[0], b.layers[0], f"backbone D {D} admitted first-layer cache")
    _backbone_truth(m, x2, cu2, f"backbone D {D} packed admission", y2)
    toks = torch.randn(6, 5, D, generator=torch.Generator().manual_seed(6)).to(dev)
    with torch.no_grad():
        for i in range(5):
            ya, yb = m.step(toks[:, i:i + 1], a), m.step(toks[:, i:i + 1], b)
            assert torch.isfinite(ya).all()
            _act(ya, yb, yb.double(), f"backbone D {D} step {i} vs the left-padded cache")


# ---------------------------------------------------------------------------------------------- 7. launches
def test_launch_counts():
    dev = _dev()
    H = _H()
    D, lcap = 16, 4096
    m = _backbone(D, lcap)
    lengths = [1 + (37 * i) % 1024 for i in range(20)] + [1025 + i for i in range(10)] + [3000]
    cu = _cu(lengths)
    x = torch.randn(cu[-1], D, generator=torch.Generator().manual_seed(6)).to(dev)
    cut = torch.tensor(cu)
    with torch.no_grad():
        m(x, cu_seqlens=cut)                                     # warm: workspaces, twiddles
        H._lib.profile_begin()
        m(x, cu_seqlens=cut)
        fwd = {k: v[1] for k, v in H._lib.profile_end().items()}
        c = m.allocate_decode_cache(len(lengths), lcap)
        H._lib.profile_begin()
        m.prefill(x, c, cu_seqlens=cut)
        pre = {k: v[1] for k, v in H._lib.profile_end().items()}
        c.release([0, 1])
        H._lib.profile_begin()
        m.admit(x[:cu[2]], c, [0, 1], cu_seqlens=torch.tensor(cu[:3]))
        adm = {k: v[1] for k, v in H._lib.profile_end().items()}
    n_layer, nb = 2, 3
    assert pre["decode_hist"] == n_layer and adm["decode_hist"] == n_layer, (pre, adm)
    for k in ("col_fwd<gate>", "col_inv<conv_fwd>", "row_pass<conv_fwd>"):
        assert pre[k] == fwd[k] == n_layer * nb, (k, pre, fwd)
        assert adm[k] == n_layer, (k, adm)                 # both admitted prompts sit in one bucket
    proj = sum(v for k, v in pre.items() if k.startswith("proj_gemm"))
    assert proj <= sum(v for k, v in fwd.items() if k.startswith("proj_gemm")), (pre, fwd)


# ---------------------------------------------------------------------------------------------- 8. Mlp rounding
@pytest.mark.parametrize("n", [4097, 4098, 4099, 5, 1030])
@pytest.mark.parametrize("batch", [1, 2])
def test_mlp_rounded_rows_keep_their_bits(n, batch):
    dev = _dev()
    H = _H()
    D = 64
    torch.manual_seed(n)
    mlp = H.Mlp(D, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh")).to(dev)
    x = torch.randn(batch, n, D, device=dev)
    with torch.no_grad():
        y = mlp(x)
        ref = H.ops.MlpFn.apply(x, mlp.fc1.weight, mlp.fc1.bias, mlp.fc2.weight, mlp.fc2.bias, mlp.approximate)
    assert torch.equal(y, ref)
    with torch.no_grad():
        y2 = mlp(x[0])                                          # (n, D): the packed layout
    assert torch.equal(y2, ref[0] if batch == 1 else H.ops.MlpFn.apply(x[:1], mlp.fc1.weight, mlp.fc1.bias,
                                                                        mlp.fc2.weight, mlp.fc2.bias, mlp.approximate)[0])
