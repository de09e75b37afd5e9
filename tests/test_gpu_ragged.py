"""Left-padded prefill of prompts of different lengths (HyenaOperator.prefill / forward / extend with ``lengths``,
hyena_b200_core_fwd_rows, hyena_b200_decode_hist_rows; DESIGN.md section 4.14).  Truth: the fp64 oracle on each row's
UNPADDED tokens.  Tolerance policy: tests/parity_util.py."""
from functools import partial

import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_widths import NANS, _poison

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _make(D, l_max, order=2, seed=0):
    """(operator on the GPU, oracle parameters) with the same weights and a non-zero in_proj bias."""
    H = _H()
    g = torch.Generator().manual_seed(seed)
    P = O.init_params(D, l_max, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    P["in_proj.bias"] = 0.02 * torch.randn(P["in_proj.bias"].shape, generator=g)
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = H.HyenaOperator(D, l_max, order=order, emb_dim=5, w=10.0)
    op.load_state_dict(sd)
    return op.to(_dev()), P


def _padded(B, P, D, lengths, seed=0, pad_seed=None, fill=None):
    """u (B, P, D) on the CPU: row b's real tokens at [P - lengths[b], P), random pads (pad_seed) before them, or pads
    filled with ``fill``: one of the NaN encodings of tests/test_gpu_widths.NANS or "inf" (random signs)."""
    u = O.nucleotide_activations(B, P, D, seed=2222 + seed)[0]
    g = torch.Generator().manual_seed(1000 + (seed if pad_seed is None else pad_seed))
    for b, n in enumerate(lengths):
        u[b, :P - n] = 3.0 * torch.randn(P - n, D, generator=g) if fill is None else _poison(u[b, :P - n], fill, g)
    return u


# non-finite pad fills: the outputs at real positions and the cache must not see them
PAD_FILLS = [*NANS, "inf"]


def _row_truth(u_row, P):
    """fp32 and fp64 oracle outputs of one unpadded row (1, n, D)."""
    return O.hyena_operator(u_row, P), O.hyena_operator(u_row.double(), O.to_dtype(P, torch.float64))


def _check_rows(y, u, lengths, P, op, tag):
    """Each row's real outputs against the oracle on its unpadded tokens; pad outputs are exactly out_proj.bias."""
    L = u.shape[1]
    bias = op.out_proj.bias.detach().cpu()
    for b, n in enumerate(lengths):
        s = L - n
        r32, r64 = _row_truth(u[b:b + 1, s:], P)
        PU.check(y[b:b + 1, s:].cpu(), r32, f"{tag} row {b} length {n}", ref64=r64)
        if s > 0:
            assert torch.equal(y[b, :s].cpu(), bias.expand(s, -1)), f"{tag} row {b}: pad outputs are not out_proj.bias"


# ---------------------------------------------------------------------------------------------- 1. pad independence
@pytest.mark.parametrize("order", [2, 3])
def test_operator_pad_independence_bitwise(order):
    dev = _dev()
    B, D, P = 4, 32, 1500
    lengths = [1500, 1, 731, 2]
    op, _ = _make(D, 2048, order)
    outs = []
    for pad_seed in (1, 2):
        u = _padded(B, P, D, lengths, pad_seed=pad_seed).to(dev)
        c = op.allocate_decode_cache(B, 2048)
        with torch.no_grad():
            y = op.prefill(u, c, lengths=lengths)
        outs.append((y, c))
    (ya, ca), (yb, cb) = outs
    assert torch.equal(ya, yb)            # the pad outputs are out_proj.bias in both
    assert torch.equal(ca.h, cb.h) and torch.equal(ca.tail, cb.tail)
    assert ca.start == tuple(P - n for n in lengths) and ca.lengths == tuple(lengths)
    for b, n in enumerate(lengths):
        assert not ca.h[:, b, :, :P - n].any()
    # NaN and +-inf pads: the same bits at the real positions and in the cache
    for fill in PAD_FILLS:
        u = _padded(B, P, D, lengths, fill=fill).to(dev)
        c = op.allocate_decode_cache(B, 2048)
        with torch.no_grad():
            y = op.prefill(u, c, lengths=lengths)
        for b, n in enumerate(lengths):
            assert torch.equal(y[b, P - n:], ya[b, P - n:]), f"{fill} pads: row {b}"
        assert torch.equal(c.h, ca.h) and torch.equal(c.tail, ca.tail), f"{fill} pads: cache"


def test_block_and_backbone_pad_independence_bitwise():
    H = _H()
    dev = _dev()
    B, D, P = 3, 32, 1100
    lengths = [1100, 3, 517]
    torch.manual_seed(0)
    block = H.Block(D, mixer_cls=partial(H.HyenaOperator, l_max=2048, emb_dim=5, w=10.0),
                    mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
    torch.manual_seed(1)
    bb = H.Backbone(D, 3, partial(H.HyenaOperator, l_max=2048, emb_dim=5, w=10.0),
                    mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
    res = {}
    for pad_seed in (1, 2, *PAD_FILLS):   # random pads, then NaN and +-inf pads
        fill = pad_seed if pad_seed in PAD_FILLS else None
        u = _padded(B, P, D, lengths, pad_seed=None if fill else pad_seed, fill=fill).to(dev)
        cb, cs = block.mixer.allocate_decode_cache(B, 2048), bb.allocate_decode_cache(B, 2048)
        with torch.no_grad():
            hb, rb = block.prefill(u, None, cb, lengths=lengths)
            hf, rf = block(u, lengths=lengths)
            ys = bb.prefill(u, cs, lengths=lengths)
            yf = bb(u, lengths=lengths)
        res[pad_seed] = (hb, rb, hf, rf, cb, ys, yf, cs)
    a = res[1]
    for key in (2, *PAD_FILLS):           # real positions only: with NaN pads the pad outputs of a block may be NaN
        b = res[key]
        for i, n in enumerate(lengths):
            s = P - n
            for j in (0, 1, 2, 3, 5, 6):
                assert torch.equal(a[j][i, s:], b[j][i, s:]), f"pads {key}: output {j} row {i}"
        for ca, cb_ in ((a[4], b[4]),) + tuple(zip(a[7].layers, b[7].layers)):
            assert torch.equal(ca.h, cb_.h) and torch.equal(ca.tail, cb_.tail), f"pads {key}: cache"
    assert torch.equal(a[0], a[2]) and torch.equal(a[5], a[6])          # forward(lengths) == prefill(lengths)
    assert a[7].start == tuple(P - n for n in lengths) and a[7].lengths == tuple(lengths)


# ---------------------------------------------------------------------------------------------- 2. arithmetic unchanged
@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("P", [1024, 1023, 4100])
def test_full_length_rows_are_plain_prefill_bits(order, P):
    dev = _dev()
    B, D = 4, 32
    lengths = [P, 5, P, 1]
    op, _ = _make(D, 8192, order)
    u = _padded(B, P, D, lengths).to(dev)
    cr, cp = op.allocate_decode_cache(B, 8192), op.allocate_decode_cache(B, 8192)
    with torch.no_grad():
        yr = op.prefill(u, cr, lengths=lengths)
        yp = op.prefill(u, cp)
    for b in (0, 2):
        assert torch.equal(yr[b], yp[b]), f"row {b}: max diff {(yr[b] - yp[b]).abs().max().item():.3e}"
        assert torch.equal(cr.h[:, b], cp.h[:, b]) and torch.equal(cr.tail[b], cp.tail[b])


# ---------------------------------------------------------------------------------------------- 3. per-row fp64 truth
def _exact_workspace(H, G):
    def ws(B, D, L, backward, device):
        n = int(H._lib.lib().hyena_b200_workspace_min_bytes(B, D, L, int(backward))) * G
        return torch.empty(n, dtype=torch.uint8, device=device)
    return ws


@pytest.mark.parametrize("P,lengths,D,path", [
    (1023, [1023, 1, 2, 3], 16, "staged"),            # odd P: register path, vec = 0
    (1024, [1024, 517, 2, 1], 16, "staged"),
    (1022, [1022, 517, 2, 1], 16, "register"),        # P % 4 == 2: register path with float2 accesses, LOGM1 of 1024
    (1025, [1025, 1024, 3, 999], 16, "staged"),
    (4096, [4096, 4095, 1, 2], 16, "groups"),         # G = 3 channels per launch: c0 > 0 and a ragged last group
    (65535, [65535, 65535 - 12345, 1, 77], 4, "staged"),
    (65536, [65536, 3, 65535, 40001], 4, "staged"),
    (65534, [65534, 3, 65533, 40001], 4, "register"),  # the same at the LOGM1 of 65536
    (65537, [65537, 2, 65536, 333], 4, "staged"),
])
def test_rows_against_fp64_truth(monkeypatch, P, lengths, D, path):
    H = _H()
    dev = _dev()
    if path == "groups":
        monkeypatch.setattr(H.ops, "workspace", _exact_workspace(H, 3))
    op, Pp = _make(D, P)
    u = _padded(len(lengths), P, D, lengths)
    with torch.no_grad():
        y = op.prefill(u.to(dev), op.allocate_decode_cache(len(lengths), P), lengths=lengths)
    _check_rows(y, u, lengths, Pp, op, f"ragged prefill P={P} {path}")


def test_order3_rows_against_fp64_truth():
    dev = _dev()
    lengths, P = [1500, 1, 2, 3, 1001], 1500
    op, Pp = _make(16, 2048, order=3)
    u = _padded(len(lengths), P, 16, lengths)
    with torch.no_grad():
        y = op.prefill(u.to(dev), op.allocate_decode_cache(len(lengths), 2048), lengths=lengths)
    _check_rows(y, u, lengths, Pp, op, "ragged prefill order 3")


def test_unaligned_operands_register_path():
    """core_forward with p at a 4-byte offset (vec = 0, no staging) and a channel group cut, on left-padded rows."""
    H = _H()
    dev = _dev()
    D, P = 8, 2048
    lengths = [2048, 1, 2, 1500]
    op, Pp = _make(D, P)
    u = _padded(len(lengths), P, D, lengths)
    with torch.no_grad():
        y_ref = op.forward(u.to(dev), lengths=lengths)
        ud = u.to(dev)
        p = H.ops.proj_gemm(ud.contiguous(), 0, op.in_proj.weight.contiguous(), False, 0)
        buf = torch.empty(p.numel() + 1, device=dev)
        pu = buf[1:].view(p.shape)
        pu.copy_(p)
        k = op.filter_fn.filter_channel_major(P)
        rs = torch.tensor([P - n for n in lengths], dtype=torch.int32, device=dev)
        args = (op.in_proj.bias.contiguous(), op.short_filter.weight.reshape(3 * D, -1).contiguous(),
                op.short_filter.bias.contiguous(), H.ops.filter_spectrum(k), op.filter_fn.bias.contiguous(), False, rs)
        y_al = H.ops.core_forward(p, *args)[0]
        y_un = H.ops.core_forward(pu, *args)[0]
        y = H.ops.proj_gemm(y_un, 1, op.out_proj.weight.contiguous(), False, 1, bias=op.out_proj.bias.contiguous())
    _check_rows(y, u, lengths, Pp, op, "ragged core 4-byte offset")
    for b, n in enumerate(lengths):
        assert not y_un[b, :, :P - n].any() and not y_al[b, :, :P - n].any()
    PU.check(y_ref, y, "ragged forward vs unaligned core")


def test_full_length_2_20():
    dev = _dev()
    P = 1 << 20
    lengths = [P, P - 12345]
    op, Pp = _make(4, P)
    u = _padded(2, P, 4, lengths)
    with torch.no_grad():
        y = op.prefill(u.to(dev), op.allocate_decode_cache(2, P), lengths=lengths)
    _check_rows(y, u, lengths, Pp, op, "ragged prefill 2^20")


# ---------------------------------------------------------------------------------------------- 4. after the prefill
def _continued_truth(u, cont, lengths, Pp):
    """Per row: the oracle on [real prompt tokens, continuation] -> (fp32, fp64) outputs of the continuation."""
    P, n = u.shape[1], cont.shape[1]
    out = []
    for b, ln in enumerate(lengths):
        seq = torch.cat([u[b:b + 1, P - ln:], cont[b:b + 1]], dim=1)
        r32, r64 = _row_truth(seq, Pp)
        out.append((r32[:, -n:], r64[:, -n:]))
    return out


def _check_cont(y, truth, tag):
    for b, (r32, r64) in enumerate(truth):
        PU.check(y[b:b + 1].cpu(), r32, f"{tag} row {b}", ref64=r64)


@pytest.mark.parametrize("order", [2, 3])
def test_steps_extend_and_graph_after_ragged_prefill(order):
    H = _H()
    dev = _dev()
    B, D, P, N = 3, 16, 700, 40
    lengths = [700, 1, 333]
    lcap = 2048
    op, Pp = _make(D, lcap, order)
    u = _padded(B, P, D, lengths)
    cont = O.nucleotide_activations(B, 3 * N, D, seed=77)[0]
    truth = _continued_truth(u, cont, lengths, Pp)
    caches = [op.allocate_decode_cache(B, lcap) for _ in range(4)]
    ud, cd = u.to(dev), cont.to(dev)
    with torch.no_grad():
        for c in caches:
            op.prefill(ud, c, lengths=lengths)
        ys = torch.cat([op.step(cd[:, i:i + 1], caches[0]) for i in range(3 * N)], 1)
        ye_direct = op._extend(cd, caches[1], H.ops.decode_extend_direct)
        ye_fft = op._extend(cd, caches[2], H.ops.decode_extend_fft)
        g = op.capture_step(caches[3], B)
        yg = torch.cat([g.step(cd[:, i:i + 1]).clone() for i in range(3 * N)], 1)
    assert torch.equal(ys, yg)                      # graph replays: the bits of eager steps on the same (plain) route
    all_truth = [(r32, r64) for r32, r64 in truth]
    _check_cont(ys, all_truth, f"order {order} steps after ragged prefill")
    _check_cont(ye_direct, all_truth, f"order {order} extend direct after ragged prefill")
    _check_cont(ye_fft, all_truth, f"order {order} extend fft after ragged prefill")
    assert caches[0].lengths == tuple(n + 3 * N for n in lengths)


def test_windowed_steps_after_ragged_prefill():
    H = _H()
    dev = _dev()
    B, D = 3, 8
    P = H.ops.WINDOW_MIN_T + 4
    N = H.ops.WINDOW_AFTER_STEPS + 24
    lengths = [P, 2, P - 40000]
    op, Pp = _make(D, P + N)
    u = _padded(B, P, D, lengths)
    cont = O.nucleotide_activations(B, N, D, seed=78)[0]
    c = op.allocate_decode_cache(B, P + N)
    with torch.no_grad():
        op.prefill(u.to(dev), c, lengths=lengths)
        ys = torch.cat([op.step(cont[:, i:i + 1].to(dev), c) for i in range(N)], 1)
    assert c.win_wc > 0                              # the window opened
    _check_cont(ys, _continued_truth(u, cont, lengths, Pp), "windowed steps after ragged prefill")


def test_fork_and_select_after_ragged_prefill():
    dev = _dev()
    B, D, P, N = 3, 16, 901, 24
    lengths = [901, 5, 450]
    op, Pp = _make(D, 2048)
    u = _padded(B, P, D, lengths)
    cont = O.nucleotide_activations(3, N, D, seed=79)[0]
    c = op.allocate_decode_cache(B, 2048)
    with torch.no_grad():
        op.prefill(u.to(dev), c, lengths=lengths)
        br = c.fork([2, 0, 2], horizon=64)
        assert br.start == (P - 450, P - 901, P - 450) and br.lengths == (450, 901, 450)
        sel = br.select([1, 0])
        assert sel.start == (P - 901, P - 450)
        ys = torch.cat([op.step(cont[:, i:i + 1].to(dev), br) for i in range(N)], 1)
        yl = torch.cat([op.step(cont[:2, i:i + 1].to(dev), sel) for i in range(N)], 1)
    rows = [2, 0, 2]
    t_br = _continued_truth(u[rows], cont, [lengths[r] for r in rows], Pp)
    _check_cont(ys, t_br, "branch steps after ragged prefill")
    t_sel = _continued_truth(u[[0, 2]], cont[:2], [lengths[0], lengths[2]], Pp)
    _check_cont(yl, t_sel, "selected branch steps after ragged prefill")


# ---------------------------------------------------------------------------------------------- 5. forward(lengths)
@pytest.mark.parametrize("order", [2, 3])
def test_forward_lengths_is_prefill_and_inference_only(order):
    H = _H()
    dev = _dev()
    lengths, P = [800, 17, 1], 800
    op, _ = _make(16, 1024, order)
    u = _padded(3, P, 16, lengths).to(dev)
    with torch.no_grad():
        yf = op(u, lengths=lengths)
        yp = op.prefill(u, op.allocate_decode_cache(3, 1024), lengths=torch.tensor(lengths))
        yc = op(u, inference_params=op.allocate_decode_cache(3, 1024), lengths=lengths)
    assert torch.equal(yf, yp) and torch.equal(yf, yc)
    n0 = H.launch_count()
    with pytest.raises(H.HyenaB200Error, match="pad them on the right"):
        op(u, lengths=lengths)
    with pytest.raises(H.HyenaB200Error, match="pad them on the right"):
        op(u.requires_grad_(True), lengths=lengths)
    assert H.launch_count() == n0


# ---------------------------------------------------------------------------------------------- 6. right padding trains
def test_right_padded_training_gradients_match_unpadded_truth():
    """The claim of forward's error message: with rows padded on the right and the loss on real positions only, the
    parameter gradients are the unpadded rows' (causal operator: pads only follow the real positions)."""
    dev = _dev()
    D, L = 16, 1200
    lengths = [1200, 700, 3]
    op, Pp = _make(D, L)
    u = O.nucleotide_activations(3, L, D, seed=5)[0]
    dy = torch.randn(3, L, D, generator=torch.Generator().manual_seed(6))
    for b, n in enumerate(lengths):
        u[b, n:] = 0.0
        dy[b, n:] = 0.0
    y = op(u.to(dev).requires_grad_(True))
    y.backward(dy.to(dev))
    got = {k: p.grad for k, p in op.named_parameters() if p.grad is not None}
    sums32, sums64 = {}, {}
    for b, n in enumerate(lengths):
        for dt, sums in ((torch.float32, sums32), (torch.float64, sums64)):
            _, _, g = O.operator_fwd_bwd(u[b:b + 1, :n].to(dt), O.to_dtype(Pp, dt), dy[b:b + 1, :n].to(dt))
            for k, v in g.items():
                sums[k] = sums.get(k, 0) + v
    assert len(sums32) == 15
    for k in sums32:
        PU.check(got[k].reshape(sums32[k].shape), sums32[k], f"right-padded grad {k}", ref64=sums64[k],
                 param_grad=True)


# ---------------------------------------------------------------------------------------------- 7. launches and kinds
@pytest.mark.parametrize("order", [2, 3])
def test_launch_counts_and_kinds(order):
    H = _H()
    dev = _dev()
    lengths, P = [1024, 9], 1024
    op, _ = _make(16, 2048, order)
    u = _padded(2, P, 16, lengths).to(dev)
    prof = {}
    for how in ("plain", "rows"):
        c = op.allocate_decode_cache(2, 2048)
        torch.cuda.synchronize()
        H._lib.profile_begin()
        n0 = H.launch_count()
        with torch.no_grad():
            op.prefill(u, c, lengths=lengths if how == "rows" else None)
        torch.cuda.synchronize()
        n = H.launch_count() - n0
        prof[how] = ({k: v[1] for k, v in H._lib.profile_end().items()}, n)
    (pk, pn), (rk, rn) = prof["plain"], prof["rows"]
    assert set(rk) <= set(pk)                          # no kind of its own
    assert rk["decode_hist"] == 1
    if order == 2:
        assert rk["col_fwd<gate>"] == rk["row_pass<conv_fwd>"] == rk["col_inv<conv_fwd>"] == 1
        # the plain prefill recomputes in_proj for the history: one projection GEMM call more
        assert rk["proj_gemm"] == pk["proj_gemm"] - 1
        same = [k for k in pk if k not in ("proj_gemm", "proj_prep")]
    else:
        same = list(pk)
        assert rn == pn
    for kind in same:
        assert rk.get(kind) == pk.get(kind), kind
