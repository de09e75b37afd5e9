"""A 16-bit decode history (DecodeCache history_dtype = torch.float16 / torch.bfloat16, DESIGN.md section 4.16) on the GPU.

The contract: the cache stores g^_o = round-to-nearest-even(g_o), g_o computed in fp32 exactly as for an fp32 cache, and
every route computes
    out_o[t] = sum_{s<=t} k_o[t-s] g^_o[s] + bias_o g^_o[t]
with fp32 arithmetic.  The tests check it four ways:
  * state bits: prefill (plain and left-padded) and admit store exactly the fp32 cache's history rounded to the 16-bit type
    and return the fp32 forward's bits; for order 2 the steps fed the same inputs keep that identity;
  * kernel bits: a dot launch over a 16-bit history gives the bits of the fp32 kernel over the same values widened into an
    fp32 twin cache, for every decode_dot_kernel<BG, R>, decode_dot_dev_kernel<BG> and decode_ext_dot_kernel<BG, NT>;
  * route results: every route's y_pre = out_{O-2} * x_0 against an fp64 recomputation from the cache's own stored g^
    (read back, widened, summed with the cache's own k and bias) under tests/parity_util.check;
  * isolation and the end-to-end error against an fp32 cache, with a bound derived from the type's unit roundoff.
"""
import math
from functools import partial

import pytest
import torch
import torch.nn.functional as F

from tests import parity_util as PU
from tests.test_gpu_decode_paths import _dev, _H, _input, _operator, _params

gpu = pytest.mark.gpu
HALF = [torch.float16, torch.bfloat16]
IDS = ["fp16", "bf16"]
UNIT_ROUNDOFF = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


# ------------------------------------------------------------------------------------------ helpers
def _setup(D, L, B, order, seed, dtype):
    P = _params(D, L, order, seed)
    op = _operator(P, D, L, order)
    u = _input(B, L, D, seed).to(_dev())
    return op, u, op.allocate_decode_cache(B, L, history_dtype=dtype)


def _taps(c, o, L):
    """(k (D, L) taps 0..L-1, bias (D,)) of recurrence o from the cache's reversed filter, in fp64."""
    D, O, ld = c.d_model, c.order, (c.lcap + 3) // 4 * 4             # a branch reads its parent's filter rows
    k = c.k[:(O - 1) * D * ld].view(D, O - 1, ld)[:, o, ld - L:].flip(-1).double()
    return k, c.bias.view(D, O - 1)[:, o].double()


def _conv64(g, k):
    """Causal convolution of g (R, D, L) with k (D, L) in fp64 -> (R, D, L)."""
    L = g.shape[-1]
    n = 1 << (2 * L - 1).bit_length()
    return torch.fft.irfft(torch.fft.rfft(g, n=n) * torch.fft.rfft(k, n=n), n=n)[..., :L]


def _ref_out(c, o, hist, t0, t1):
    """fp64 out_o at positions [t0, t1) from the stored history hist (R, D, >= t1) of recurrence o."""
    g = hist[..., :t1].double()
    k, b = _taps(c, o, t1)
    return _conv64(g, k)[..., t0:t1] + b[:, None] * g[..., t0:t1]


def _check(y_pre, x0, c, t0, t1, what, hist=None, rows=None):
    """y_pre (B, D, n) of positions [t0, t1) against out_{O-2} * x_0 recomputed in fp64 from the cache's stored g^ (of the
    batch rows ``rows`` only, when given)."""
    o = c.order - 2
    hist = c.h[o] if hist is None else hist
    ref = _ref_out(c, o, hist, t0, t1) * x0.double()
    if rows is not None:
        y_pre, ref = y_pre[rows], ref[rows]
    PU.check(y_pre, ref.float(), what, ref64=ref)


def _p_t(op, u_t):
    return F.linear(u_t.reshape(u_t.shape[0], -1).float(), op.in_proj.weight).contiguous()


def _steps(op, c, u, n, core=None):
    """n steps from c.t on through ops (y_pre and x_0 of each) -> (y_pre (B, D, n), x_0 (B, D, n))."""
    H = _H()
    core = core or H.ops.decode_step_auto
    ib, sw, sb = op._decode_params()
    ys, xs = [], []
    with torch.no_grad():
        for _ in range(n):
            ys.append(core(_p_t(op, u[:, c.t]), ib, sw, sb, c))
            xs.append(c.s_t[:, :c.d_model].clone())
            c.t += 1
    return torch.stack(ys, -1), torch.stack(xs, -1)


@pytest.fixture
def capture_s(monkeypatch):
    """The short-filter outputs s (B, C, n) of each extend, captured from ops.decode_extend_hist."""
    H = _H()
    got, orig = [], H.ops.decode_extend_hist

    def hist(*a):
        got.append(orig(*a))
        return got[-1]
    monkeypatch.setattr(H.ops, "decode_extend_hist", hist)
    return got


def _extend(op, c, u, n, how, got):
    H = _H()
    core = H.ops.decode_extend_direct if how == "direct" else H.ops.decode_extend_fft
    ib, sw, sb = op._decode_params()
    with torch.no_grad():
        p = H.ops.proj_gemm(u[:, c.t:c.t + n].contiguous(), 0, op.in_proj.weight.detach().contiguous(), False, 0)
        H._lib.profile_begin()
        y = core(p, ib, sw, sb, c)
        prof = H._lib.profile_end()
    assert ("decode_extend_dot" in prof) == (how == "direct"), prof
    x0 = got[-1][:, :c.d_model]
    c.t += n
    return y, x0


# ------------------------------------------------------------------------------------------ 1. state bits
@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("D", [1, 3, 100, 256])
def test_state_bits(dtype, order, D):
    """prefill, left-padded prefill and admit store the fp32 cache's history rounded to the type, bit for bit, and return
    the fp32 forward's bits; for order 2 steps fed the same inputs keep the identity (g_0 does not read the history)."""
    B, P0, n = 3, 1021, 6
    L = P0 + n
    op, u, c16 = _setup(D, L, B, order, 7 * D + order, dtype)
    c32 = op.allocate_decode_cache(B, L)
    with torch.no_grad():
        assert torch.equal(op.prefill(u[:, :P0], c16), op.prefill(u[:, :P0], c32))
        assert torch.equal(c16.h, c32.h.to(dtype)) and torch.equal(c16.tail, c32.tail)
        assert c16.history_dtype == dtype and c16.h.dtype == dtype and c16.k.dtype == torch.float32
        if order == 2:
            for i in range(P0, L):
                op.step(u[:, i:i + 1], c16)
                op.step(u[:, i:i + 1], c32)
            assert torch.equal(c16.h, c32.h.to(dtype)) and torch.equal(c16.tail, c32.tail)
        # left-padded prefill
        lengths = [P0, P0 - 5, 17][:B]
        r16, r32 = op.allocate_decode_cache(B, L, history_dtype=dtype), op.allocate_decode_cache(B, L)
        assert torch.equal(op.prefill(u[:, :P0], r16, lengths=lengths), op.prefill(u[:, :P0], r32, lengths=lengths))
        assert torch.equal(r16.h, r32.h.to(dtype)) and torch.equal(r16.tail, r32.tail)
        # admission into row 1 at the running position
        Pa = 301
        ya16 = op.admit(u[1:2, :Pa], r16, [1])
        ya32 = op.admit(u[1:2, :Pa], r32, [1])
        assert torch.equal(ya16, ya32)
        assert torch.equal(r16.h, r32.h.to(dtype)) and torch.equal(r16.tail, r32.tail)


# ------------------------------------------------------------------------------------------ 2. kernel bits
def _twin(c16, op, B, L):
    c32 = op.allocate_decode_cache(B, L)
    c32.h.copy_(c16.h.float())
    c32.tail.copy_(c16.tail)
    c32.t = c16.t
    return c32


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("B", [1, 2, 3, 5])
def test_dot_kernel_bits(dtype, B):
    """decode_dot_kernel<BG, R> (BG from B = 1, 2, 3, 5; R from t = 2045..2048), decode_dot_dev_kernel<BG> and
    decode_ext_dot_kernel<BG, NT> (NT from n = 8, 9) over a 16-bit history give the partial sums of the fp32 kernels over
    the same values widened into an fp32 twin cache, bit for bit."""
    H = _H()
    D, P0, L = 100, 2049, 2064
    op, u, c16 = _setup(D, L, B, 2, 11 * B, dtype)
    with torch.no_grad():
        op.prefill(u[:, :P0], c16)
        c32 = _twin(c16, op, B, L)
        ib, sw, sb = op._decode_params()
        for t in range(2045, 2049):
            for c in (c16, c32):
                c.t = t
            p_t = _p_t(op, u[:, t])
            for dev in (False, True):
                for c in (c16, c32):
                    saved = (c.h.clone(), c.tail.clone())
                    if dev:
                        c.sync_position()
                        H.ops.decode_step_dev(p_t, ib, sw, sb, c, L)
                    else:
                        H.ops.decode_step(p_t, ib, sw, sb, c)
                    c.h.copy_(saved[0])
                    c.tail.copy_(saved[1])
                nch = -(-t // 1024)
                assert torch.equal(c16.part[..., :nch], c32.part[..., :nch]), (t, dev)
        for t, n in [(1021, 8), (1022, 9), (2047, 9), (2040, 8)]:
            parts = []
            for c in (c16, c32):
                groups = int(H._lib.lib().hyena_b200_decode_extend_groups(B, D, t, n))
                part = torch.full((B, D, n, groups), float("nan"), device=u.device)
                H._lib.check(H.ops._decode_fn("extend_dot", c.h)(
                    H.ops._ptr(c.h[0]), H.ops._ptr(c.k), H.ops._ptr(part), groups, B, B, D, 2, 0, t, n, c.lcap,
                    H.ops._stream()))
                parts.append(part)
            assert torch.equal(parts[0], parts[1]), (t, n)


# ------------------------------------------------------------------------------------------ 3. route results
@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("D", [1, 3, 100, 256])
def test_plain_steps_and_extends(capture_s, dtype, order, D):
    """Plain steps across a chunk boundary, direct extends with n = 9 and 511 and an FFT extend with n = 512, each against
    the fp64 recomputation from the stored history."""
    B = 3 if D < 256 else 2
    P0 = 1021
    plan = [("step", 5), ("direct", 9), ("direct", 511), ("fft", 512), ("step", 3)]
    L = P0 + sum(n for _, n in plan)
    op, u, c = _setup(D, L, B, order, 13 * D + order, dtype)
    with torch.no_grad():
        op.prefill(u[:, :P0], c)
    for how, n in plan:
        t0 = c.t
        if how == "step":
            y, x0 = _steps(op, c, u, n)
        else:
            y, x0 = _extend(op, c, u, n, how, capture_s)
        _check(y, x0, c, t0, t0 + n, f"{dtype} order {order} D={D} {how} [{t0}, {t0 + n})")


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
def test_windowed_steps_long_history(dtype, order):
    """Steps at t >= 2^16: the window opens after WINDOW_AFTER_STEPS plain steps (its F from the FFT of the widened
    history) and the windowed steps meet the contract."""
    H = _H()
    D, B = 3, 2
    P0 = (1 << 16) + 1
    n = H.ops.WINDOW_AFTER_STEPS + 6
    op, u, c = _setup(D, P0 + n, B, order, 5 + order, dtype)
    with torch.no_grad():
        op.prefill(u[:, :P0], c)
    y, x0 = _steps(op, c, u, n)
    assert c.win_wc > 0 and c.win_b <= c.t - 1, (c.win_b, c.win_wc)
    _check(y, x0, c, P0, P0 + n, f"{dtype} order {order} windowed")


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
def test_branches(dtype, order):
    """A fork of 3 and of 17 branches, then select, stepped on the branch route; the reference sums the parent rows'
    stored history before the base and each branch's own history after it."""
    H = _H()
    D, B, t0 = 100, 2, 1022
    L = t0 + 12
    op, u, c = _setup(D, L, B, order, 17 + order, dtype)
    with torch.no_grad():
        op.prefill(u[:, :t0], c)
    for rows in ([1, 0, 1], [i % B for i in range(17)]):
        br = c.fork(rows, horizon=8)
        assert br.h.dtype == dtype and br.f.dtype == torch.float32
        sel = [len(rows) - 1 - i for i in range(len(rows))]
        for cache, rr in ((br, rows), (br.select(sel), [rows[i] for i in sel])):
            uu = u[rr]
            y, x0 = _steps(op, cache, uu, 5, core=H.ops.decode_branch_step)
            o, b = order - 2, cache.base
            hist = torch.cat([c.h[o][rr][..., :b], cache.h[o][..., :cache.t - b]], dim=-1)
            _check(y, x0, cache, cache.t - 5, cache.t, f"{dtype} order {order} {len(rows)} branches", hist=hist)


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
def test_step_graph_bits(dtype, order):
    """StepGraph replays on a 16-bit cache are the bits of eager steps on a twin cache (outputs and stored history)."""
    H = _H()
    D, B, P0, n = 100, 3, 1019, 9
    op, u, ce = _setup(D, P0 + n, B, order, 23 + order, dtype)
    cg = op.allocate_decode_cache(B, P0 + n, history_dtype=dtype)
    with torch.no_grad():
        op.prefill(u[:, :P0], ce)
        op.prefill(u[:, :P0], cg)
        g = H.StepGraph(op, cg, B, torch.float32)
        for i in range(P0, P0 + n):
            assert torch.equal(op.step(u[:, i:i + 1], ce), g.step(u[:, i:i + 1])), i
    assert torch.equal(ce.h, cg.h) and cg.t == ce.t


@pytest.fixture
def small_windows(monkeypatch):
    """Windows of 64 positions that open after 2 steps at any history."""
    ops = _H().ops
    monkeypatch.setattr(ops, "WINDOW", 64)
    monkeypatch.setattr(ops, "WINDOW_MIN_T", 0)
    monkeypatch.setattr(ops, "WINDOW_AFTER_STEPS", 2)


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("order", [2, 3])
def test_serving(small_windows, dtype, order):
    """admit, release and compact on a 16-bit cache (the window kept and closed by a compaction): the steps after each
    meet the contract on the cache's shifted history."""
    D, B = 100, 4
    L = 1500
    op, u, c = _setup(D, L, B, order, 29 + order, dtype)
    with torch.no_grad():
        op.prefill(u[:, :300], c, lengths=[300, 200, 150, 120])
    y, x0 = _steps(op, c, u, 4)                                      # opens a window
    _check(y, x0, c, c.t - 4, c.t, f"{dtype} serving steps")
    assert c.win_wc > 0
    with torch.no_grad():
        op.admit(u[2:3, :90], c, [2])                                  # into an open window
    y, x0 = _steps(op, c, u, 3)
    _check(y, x0, c, c.t - 3, c.t, f"{dtype} after admit")
    c.release([0])
    win = (c.win_b, c.win_wc)
    m = c.compact()                                                  # row 0 freed: the shift keeps the window
    assert m > 0 and c.win_wc == win[1], (m, win, c.win_b, c.win_wc)
    y, x0 = _steps(op, c, u, 3)
    # the kept window's F of the released row 0 still holds the history the shift dropped: its outputs are not checked
    _check(y, x0, c, c.t - 3, c.t, f"{dtype} after compact, window kept", rows=[1, 2, 3])
    c.release([1, 2, 3])
    with torch.no_grad():
        op.admit(u[1:2, :4], c, [1])
    m = c.compact()                                                  # moves past the window base: it closes
    assert m > 0 and c.win_wc == 0, (m, c.win_b, c.win_wc)
    y, x0 = _steps(op, c, u, 4)
    _check(y, x0, c, c.t - 4, c.t, f"{dtype} after compact, window closed")


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
def test_large_batch(capture_s, dtype):
    """B * D = 257 * 256 > 65535 rows on the history kernels' x grid, steps and a direct extend."""
    D, B, P0 = 256, 257, 37
    op, u, c = _setup(D, P0 + 12, B, 2, 31, dtype)
    with torch.no_grad():
        op.prefill(u[:, :P0], c)
    y, x0 = _steps(op, c, u, 3)
    _check(y, x0, c, P0, P0 + 3, f"{dtype} B*D > 65535 steps")
    y, x0 = _extend(op, c, u, 9, "direct", capture_s)
    _check(y, x0, c, P0 + 3, P0 + 12, f"{dtype} B*D > 65535 extend")


# ------------------------------------------------------------------------------------------ 4. isolation
@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
@pytest.mark.parametrize("bad", ["nan", "inf", "overflow"])
def test_row_isolation(dtype, bad):
    """A NaN, +-inf or overflowing row stays in its row: the other rows' outputs and history are the bits of a run without
    it.  "overflow" scales one row's input so that g exceeds 65504, the fp16 range: its fp16 history stores +-inf."""
    H = _H()
    D, B, P0, n = 100, 3, 1021, 4
    op, u, c = _setup(D, P0 + n + 9, B, 2, 37, dtype)
    bad_u = u.clone()
    if bad == "overflow":
        bad_u[1] *= 3e3
    else:
        bad_u[1, 500:505] = float("nan") if bad == "nan" else float("inf")
    clean = op.allocate_decode_cache(B, P0 + n + 9, history_dtype=dtype)
    with torch.no_grad():
        ys = [op.prefill(bad_u[:, :P0], c), op.step(bad_u[:, P0:P0 + 1], c), op.extend(bad_u[:, P0 + 1:P0 + 10], c)]
        yc = [op.prefill(u[:, :P0], clean), op.step(u[:, P0:P0 + 1], clean), op.extend(u[:, P0 + 1:P0 + 10], clean)]
    keep = [0, 2]
    for a, b in zip(ys, yc):
        assert torch.equal(a[keep], b[keep])
    assert torch.equal(c.h[:, keep], clean.h[:, keep])
    if bad == "overflow":
        if dtype == torch.float16:
            assert torch.isinf(c.h[0, 1]).any(), "the scaled row should overflow the fp16 history"
        else:
            assert torch.isfinite(c.h[0, 1]).all(), "bf16 has the fp32 exponent range"


# ------------------------------------------------------------------------------------------ 5. end to end against fp32
def _backbone(D, L, seed):
    H = _H()
    torch.manual_seed(seed)
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh"))
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, H.HyenaOperator):
                mod.in_proj.bias.normal_(0, 0.02)
    return m.to(_dev())


def _condition(c, t0, t1):
    """kappa = || u-worst-case perturbation of the layer's long sum || / || the sum ||, from an fp32 cache's history:
    ||(|k| * |g| + |bias| |g|)[t0, t1)|| / ||(k * g + bias g)[t0, t1)|| (recurrence 0, * the causal convolution)."""
    g = c.h[0][..., :t1].double()
    k, b = _taps(c, 0, t1)
    out = _conv64(g, k)[..., t0:t1] + b[:, None] * g[..., t0:t1]
    worst = _conv64(g.abs(), k.abs())[..., t0:t1] + b.abs()[:, None] * g[..., t0:t1].abs()
    return float(worst.norm() / out.norm())


@gpu
@pytest.mark.parametrize("dtype", HALF, ids=IDS)
def test_backbone_end_to_end(dtype):
    """A 2-layer Backbone with Mlp at D = 256 prefilled to 2^17 and stepped 256 positions with a 16-bit and an fp32 cache.

    Bound.  The two runs differ only by the rounding of the stored history: g^ = g (1 + e), |e| <= u (u = 2^-11 for fp16,
    2^-8 for bf16).  To first order, layer l's long sum out_l = k * g^ + bias g^ moves by at most u (|k| * |g| + |bias| |g|)
    elementwise, a normwise relative change of at most u kappa_l, with kappa_l the ratio of those two norms computed from
    the fp32 cache over the stepped positions (_condition).  y_pre = out x_0 and out_proj are linear in out, the residual
    add and the LayerNorm (whose mean and scale are set by the whole residual stream) leave a relative change of the same
    first order, and the gated MLP and layer 2 carry layer 1's change on: the backbone's output moves by at most about
    sum_l u kappa_l.  The test allows twice that, 2 u sum_l kappa_l, for the second-order terms and the changed inputs of
    layer 2, and prints the measured normwise error (recorded in DESIGN.md section 4.16)."""
    D, T, n = 256, 1 << 17, 256
    m = _backbone(D, T + n, 41)
    x = _input(1, T + n, D, 41).to(_dev())
    outs = {}
    for hd in (torch.float32, dtype):
        c = m.allocate_decode_cache(1, T + n, history_dtype=hd)
        assert c.history_dtype == hd
        with torch.no_grad():
            y0 = m.prefill(x[:, :T], c)
            ys = [m.step(x[:, i:i + 1], c) for i in range(T, T + n)]
        outs[hd] = (y0, torch.cat(ys, dim=1), c)
    assert torch.equal(outs[dtype][0], outs[torch.float32][0])     # prefill returns the fp32 forward's bits
    c32 = outs[torch.float32][2]
    kappa = [_condition(c32.for_module(layer.mixer), T, T + n) for layer in m.layers]
    bound = 2 * UNIT_ROUNDOFF[dtype] * sum(kappa)
    y16, y32 = outs[dtype][1].double(), outs[torch.float32][1].double()
    err = float((y16 - y32).norm() / y32.norm())
    print(f"\n{dtype}: normwise relative error of 256 steps after 2^17 = {err:.3e}; kappa = "
          f"{', '.join(f'{k:.2f}' for k in kappa)}; bound 2 u sum kappa = {bound:.3e}; "
          f"nbytes {outs[dtype][2].nbytes} vs {c32.nbytes}")
    assert math.isfinite(err) and err <= bound, (err, bound, kappa)
    hist = sum(cl.h.numel() for cl in c32.layers)
    assert c32.nbytes - outs[dtype][2].nbytes == 2 * hist and outs[dtype][2].history_dtype == dtype
