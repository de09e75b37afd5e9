"""Training on left-padded batches (``forward(u, mask=...)`` of HyenaOperator, Block and Backbone;
hyena_b200_core_bwd_rows; DESIGN.md section 4.17).  Truth: the oracle on each row's UNPADDED tokens in fp32 and fp64, the
parameter gradients summed over the rows (tests/test_ragged_train_cpu.row_truth).  Tolerance policy:
tests/parity_util.py."""
from functools import partial

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_ragged import PAD_FILLS, _exact_workspace, _make, _padded
from tests.test_ragged_train_cpu import row_truth

pytestmark = pytest.mark.gpu

SKIP = ("filter_fn.pos_emb.z", "filter_fn.pos_emb.t", "filter_fn.modulation.deltas")


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _mask(lengths, P):
    return torch.stack([torch.arange(P) >= P - n for n in lengths])


def _dy(u, lengths, seed=6, pads="zero"):
    """Upstream gradient: random on the real positions; at the pads zero (the loss of a padded batch) or, pads="random",
    random values of a loss that also reads the pad outputs."""
    B, P, D = u.shape
    dy = torch.randn(B, P, D, generator=torch.Generator().manual_seed(seed))
    if pads == "zero":
        for b, n in enumerate(lengths):
            dy[b, :P - n] = 0.0
    return dy


def _train(model, u, dy, mask, **kw):
    """One masked training step on the GPU -> (y, du, {parameter name: grad}) on the CPU."""
    dev = _dev()
    model.zero_grad(set_to_none=True)
    ud = u.to(dev).requires_grad_(True)
    y = model(ud, mask=mask, **kw) if mask is not None else model(ud, **kw)
    y.backward(dy.to(dev))
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu() for k, p in model.named_parameters() if p.grad is not None}
    return y.detach().cpu(), ud.grad.detach().cpu(), grads


def _check_truth(res, u, dy, lengths, Pp, op, tag):
    """Real positions against the per-row truth, all 15 parameter gradients against its sums, the pads exactly.  The
    outputs at the pads are out_proj.bias, so d out_proj.bias is the truth's plus the sum of dy over the pads; dy at the
    pads reaches no other gradient."""
    y, du, grads = res
    P = u.shape[1]
    ys32, dus32, s32 = row_truth(u, dy, lengths, Pp, torch.float32)
    ys64, dus64, s64 = row_truth(u, dy, lengths, Pp, torch.float64)
    pad_dy = sum(dy[b, :P - n].double().sum(0) for b, n in enumerate(lengths))
    s32["out_proj.bias"] = s32["out_proj.bias"] + pad_dy.float()
    s64["out_proj.bias"] = s64["out_proj.bias"] + pad_dy
    bias = op.out_proj.bias.detach().cpu()
    for b, n in enumerate(lengths):
        s = P - n
        PU.check(y[b:b + 1, s:], ys32[b], f"{tag} y row {b} length {n}", ref64=ys64[b])
        PU.check(du[b:b + 1, s:], dus32[b], f"{tag} du row {b} length {n}", ref64=dus64[b])
        if s > 0:
            assert not du[b, :s].any(), f"{tag} row {b}: du is not 0 at the pads"
            assert torch.equal(y[b, :s], bias.expand(s, -1)), f"{tag} row {b}: pad outputs are not out_proj.bias"
    assert len(s32) >= 15
    for k in s32:
        PU.check(grads[k].reshape(s32[k].shape), s32[k], f"{tag} grad {k}", ref64=s64[k], param_grad=True)


def _lengths(P):
    """1, 2 and P, and row starts at every residue mod 4 (0, P-1, P-2, 1, 2, 3)."""
    return [P, 1, 2, P - 1, P - 2, P - 3]


# ---------------------------------------------------------------------------------------------- 1. operator, per-row truth
OPERATOR_CASES = [
    (2, 1, 1023), (2, 3, 1026), (2, 100, 1024), (2, 256, 1024), (2, 256, 1023),      # odd: vec = 0; 1026: unstaged
    (3, 3, 1023), (3, 100, 1026), (3, 256, 1024),
]


def _with_dy_pads(cases):
    """Each case with dy zero at the pads (its plain id) and with dy random there (id suffix "dy_pads")."""
    ids = lambda c: "-".join(map(str, c if isinstance(c, tuple) else (c,)))
    out = []
    for c in cases:
        t = c if isinstance(c, tuple) else (c,)
        out += [pytest.param(*t, "zero", id=ids(c)), pytest.param(*t, "random", id=ids(c) + "-dy_pads")]
    return out


@pytest.mark.parametrize("order,D,P,dy_pads", _with_dy_pads(OPERATOR_CASES))
def test_operator_against_per_row_truth(order, D, P, dy_pads):
    lengths = _lengths(P)
    op, Pp = _make(D, P, order)
    u = _padded(len(lengths), P, D, lengths)
    dy = _dy(u, lengths, pads=dy_pads)
    _check_truth(_train(op, u, dy, _mask(lengths, P)), u, dy, lengths, Pp, op, f"order {order} D={D} P={P}")


# ---------------------------------------------------------------------------------------------- 2. routes
@pytest.mark.parametrize("route,dy_pads", _with_dy_pads(["fused", "library", "recompute", "batch1", "groups"]))
def test_routes_against_per_row_truth(monkeypatch, route, dy_pads):
    H = _H()
    D, P = 8, 2048
    lengths = [2048, 1, 1027, 2, 514]
    if route == "library":
        H.ops.proj_mode()
        monkeypatch.setattr(H.ops, "_proj_mode", "lt")
        assert H.ops.proj_mode() == "lt"
    elif route == "recompute":
        monkeypatch.setenv("HYENA_B200_SAVE_SPECTRUM", "0")
    elif route == "batch1":                       # B = 1 with the g spectrum saved: the batch-1 row pass of the backward
        lengths = [2048 - 777]
    elif route == "groups":                       # workspace for 3 channels: groups 3 + 3 + 2, c0 > 0, a ragged last group
        monkeypatch.setattr(H.ops, "workspace", _exact_workspace(H, 3))
    op, Pp = _make(D, P)
    u = _padded(len(lengths), P, D, lengths)
    dy = _dy(u, lengths, pads=dy_pads)
    H._lib.profile_begin()
    res = _train(op, u, dy, _mask(lengths, P))
    prof = {k: v[1] for k, v in H._lib.profile_end().items()}
    if route == "recompute":
        assert prof["col_fwd<gate>"] == 2, prof          # forward + the recomputation in the backward
    if route == "library":
        assert prof.get("short_conv_bwd") == 1, prof
    if route == "groups":
        assert prof["col_fwd<dc>"] == 3, prof
    _check_truth(res, u, dy, lengths, Pp, op, f"route {route}")


def test_long_row_2_20():
    P = 1 << 20
    lengths = [P - 777]
    op, Pp = _make(64, P)
    u = _padded(1, P, 64, lengths)
    dy = _dy(u, lengths)
    _check_truth(_train(op, u, dy, _mask(lengths, P)), u, dy, lengths, Pp, op, "2^20 start 777")


# ---------------------------------------------------------------------------------------------- 3. pad independence
# gradients summed by atomicAdd across CTAs (the fused pass-3 reductions, and d in_proj.bias derived from them): their
# summation order varies from run to run, so two identical runs can differ in the last bits
ATOMIC = ("filter_fn.bias", "short_filter.weight", "short_filter.bias", "in_proj.bias")


def _reproducible(a, b):
    """Names of the gradients two identical runs give bit for bit, atomic sums excluded."""
    return {k for k in a if torch.equal(a[k], b[k]) and not k.endswith(ATOMIC)}


def _same(ga, gb, exact, tag):
    for k in ga:
        if k in exact:
            assert torch.equal(ga[k], gb[k]), f"{tag}: grad {k} differs"
        else:
            scale = float(ga[k].abs().max())
            assert torch.allclose(ga[k], gb[k], rtol=1e-5, atol=1e-6 * max(scale, 1e-30)), f"{tag}: grad {k}"


@pytest.mark.parametrize("order", [2, 3])
def test_pad_independence(order):
    B, D, P = 4, 32, 1500
    lengths = [1500, 1, 731, 2]
    op, _ = _make(D, 2048, order)
    m = _mask(lengths, P)
    ref = None
    for fill in (1, 1, 2, *PAD_FILLS):
        u = _padded(B, P, D, lengths, pad_seed=fill if fill in (1, 2) else None,
                    fill=None if fill in (1, 2) else fill)
        y, du, g = _train(op, u, _dy(u, lengths), m)
        assert all(torch.isfinite(v).all() for v in g.values()), f"pads {fill}: non-finite gradient"
        if ref is None:
            ref, exact = (y, du, g), None
            continue
        if exact is None:                            # the same pads twice: which gradients are reproducible
            exact = _reproducible(ref[2], g)
        assert torch.equal(y, ref[0]) and torch.equal(du, ref[1]), f"pads {fill}: y / du"
        _same(ref[2], g, exact, f"pads {fill}")
    assert {"in_proj.weight", "out_proj.weight"} <= exact


# ---------------------------------------------------------------------------------------------- 4. the existing paths
@pytest.mark.parametrize("order", [2, 3])
def test_agreement_with_lengths_and_plain(order):
    dev = _dev()
    B, D, P = 3, 16, 1000
    lengths = [1000, 17, 1]
    op, _ = _make(D, 1024, order)
    u = _padded(B, P, D, lengths).to(dev)
    m = _mask(lengths, P)
    with torch.no_grad():
        yl = op(u, lengths=lengths)
        for mm in (m, m.to(dev), m.to(torch.int64)):
            assert torch.equal(op(u, mask=mm), yl)
    dy = _dy(u.cpu(), lengths)
    yg, _, _ = _train(op, u.cpu(), dy, m)
    assert torch.equal(yg, yl.cpu())                  # the differentiable route computes the same bits
    # an all-ones mask is the plain operator: y bit for bit, gradients as two plain runs agree
    full = torch.ones(B, P, dtype=torch.bool)
    dyf = torch.randn(B, P, D, generator=torch.Generator().manual_seed(9))
    y1, du1, g1 = _train(op, u.cpu(), dyf, None)
    y2, du2, g2 = _train(op, u.cpu(), dyf, None)
    ym, dum, gm = _train(op, u.cpu(), dyf, full)
    assert torch.equal(ym, y1) and torch.equal(dum, du1)
    _same(g1, gm, _reproducible(g1, g2), "all-ones mask vs plain")


# ---------------------------------------------------------------------------------------------- 5. Block and Backbone
def _backbone_truth(bb, u, dy, lengths, dtype):
    """fp32 / fp64 per-row composition of the Backbone's own parameters (O.prenorm_backbone on each unpadded row) ->
    (per-row outputs, per-row input gradients, parameter gradients summed over the rows)."""
    P = u.shape[1]
    names = [k for k, _ in bb.named_parameters() if not k.endswith(SKIP)]
    ys, dus, sums = [], [], {}
    for b, n in enumerate(lengths):
        sd = {k: v.detach().cpu().to(dtype).clone().requires_grad_(k in names) for k, v in bb.state_dict().items()}
        for i in range(len(bb.layers)):             # the three Sin modules of a filter share one freq
            for j in (3, 5):
                sd[f"layers.{i}.mixer.filter_fn.implicit_filter.{j}.freq"] = sd[f"layers.{i}.mixer.filter_fn.implicit_filter.1.freq"]
        x = u[b:b + 1, P - n:].to(dtype).clone().requires_grad_(True)
        y = O.prenorm_backbone(x, sd, len(bb.layers))
        y.backward(dy[b:b + 1, P - n:].to(dtype))
        ys.append(y.detach())
        dus.append(x.grad.detach())
        for k in names:
            sums[k] = sums.get(k, 0) + sd[k].grad
    return ys, dus, sums


@pytest.mark.parametrize("D", [3, 100, 256])
def test_backbone_against_per_row_composition(D):
    H = _H()
    dev = _dev()
    B, P = 4, 1024
    lengths = [1024, 1, 2, 513]
    torch.manual_seed(D)
    bb = H.Backbone(D, 2, partial(H.HyenaOperator, l_max=P, emb_dim=5, w=10.0),
                    mlp_cls=partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh")),
                     residual_in_fp32=True).to(dev)
    u = _padded(B, P, D, lengths)
    dy = _dy(u, lengths)
    y, du, g = _train(bb, u, dy, _mask(lengths, P))
    ys32, dus32, s32 = _backbone_truth(bb, u, dy, lengths, torch.float32)
    ys64, dus64, s64 = _backbone_truth(bb, u, dy, lengths, torch.float64)
    for b, n in enumerate(lengths):
        s = P - n
        PU.check(y[b:b + 1, s:], ys32[b], f"backbone D={D} y row {b}", ref64=ys64[b])
        PU.check(du[b:b + 1, s:], dus32[b], f"backbone D={D} du row {b}", ref64=dus64[b])
        assert not du[b, :s].any(), f"backbone D={D} row {b}: du is not 0 at the pads"
    for k in s32:
        PU.check(g[k].reshape(s32[k].shape), s32[k], f"backbone D={D} grad {k}", ref64=s64[k], param_grad=True)
    # finite pads: the same gradients (bitwise where two identical runs agree bitwise)
    _, _, g1 = _train(bb, u, dy, _mask(lengths, P))
    u2 = _padded(B, P, D, lengths, pad_seed=2)
    y2, du2, g2 = _train(bb, u2, dy, _mask(lengths, P).to(dev))
    for b, n in enumerate(lengths):
        assert torch.equal(y2[b, P - n:], y[b, P - n:]) and torch.equal(du2[b], du[b])
    _same(g, g2, _reproducible(g, g1), f"backbone D={D} pads")


def test_block_mask_matches_backbone_layer():
    """Block.forward(mask=) is the Backbone's layer: same bits as driving the block directly."""
    H = _H()
    dev = _dev()
    D, P = 16, 700
    lengths = [700, 3, 350]
    torch.manual_seed(0)
    block = H.Block(D, mixer_cls=partial(H.HyenaOperator, l_max=1024, emb_dim=5, w=10.0),
                    mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
    u = _padded(3, P, D, lengths).to(dev)
    with torch.no_grad():
        hm, rm = block(u, mask=_mask(lengths, P))
        hl, rl = block(u, lengths=lengths)
    assert torch.equal(hm, hl) and torch.equal(rm, rl)


# ---------------------------------------------------------------------------------------------- 6. launches
@pytest.mark.parametrize("order", [2, 3])
def test_launch_counts_per_kind(order):
    H = _H()
    dev = _dev()
    D, P = 16, 1024
    lengths = [1024, 9]
    op, _ = _make(D, 2048, order)
    u = _padded(2, P, D, lengths).to(dev)
    dy = _dy(u.cpu(), lengths).to(dev)
    counts = {}
    for how in ("plain", "mask", "plain"):
        ud = u.clone().requires_grad_(True)
        y = op(ud, mask=_mask(lengths, P)) if how == "mask" else op(ud)
        torch.cuda.synchronize()
        H._lib.profile_begin()
        y.backward(dy)
        torch.cuda.synchronize()
        counts[how] = {k: v[1] for k, v in H._lib.profile_end().items()}
    assert counts["mask"] == counts["plain"], (counts["mask"], counts["plain"])
