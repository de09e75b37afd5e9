"""Packed variable-length batches (``forward(u, cu_seqlens=...)`` of HyenaOperator, Block and Backbone;
hyena_b200_core_fwd_packed / core_bwd_packed / short_bwd_packed; DESIGN.md section 4.18).  Truth: the oracle on each
sequence alone, in fp32 (``ref32``) and fp64, on the device; parameter gradients are the sums over the sequences
(tests/test_varlen_cpu.seq_truth).  Tolerance policy: tests/parity_util.py."""
from functools import partial

import pytest
import torch
import torch.nn.functional as F

from tests import parity_util as PU
from tests.test_gpu_block_paths import _check_grads, _leaves, _ln_randomize
from tests.test_gpu_decode_paths import backbone_ref
from tests.test_gpu_ragged import _make
from tests.test_gpu_widths import _act
from tests.test_varlen_cpu import packed_input, seq_truth

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _train(model, u, dy, cu, **kw):
    """One packed training step -> (y, du, {parameter name: grad}) on the device."""
    dev = _dev()
    model.zero_grad(set_to_none=True)
    ud = u.to(dev).requires_grad_(True)
    y = model(ud, cu_seqlens=cu, **kw)
    y.backward(dy.to(dev))
    torch.cuda.synchronize()
    return y.detach(), ud.grad.detach(), {k: p.grad.detach() for k, p in model.named_parameters() if p.grad is not None}


def _check_truth(res, u, dy, cu, P, tag, only=None):
    """Every sequence's y and du against its own truth, every parameter gradient against the sums."""
    y, du, grads = res
    dev = _dev()
    t32 = seq_truth(u, dy, cu, P, torch.float32, dev, only)
    t64 = seq_truth(u, dy, cu, P, torch.float64, dev, only)
    for i, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        if b > a and (only is None or i in only):
            PU.check(y[a:b], t32[0][i], f"{tag} y seq {i} length {b - a}", ref64=t64[0][i])
            PU.check(du[a:b], t32[1][i], f"{tag} du seq {i} length {b - a}", ref64=t64[1][i])
    assert len(t32[2]) >= 15
    for k in t32[2]:
        PU.check(grads[k].reshape(t32[2][k].shape), t32[2][k], f"{tag} grad {k}", ref64=t64[2][k], param_grad=True)


def _edges(hi):
    """1 to 3, and both sides of every power of two from 2^10 to hi."""
    out = [1, 2, 3]
    k = 1024
    while k <= hi:
        out += [k - 1, k, k + 1] if k < hi else [k - 1, k]
        k *= 2
    return out


# ---------------------------------------------------------------------------------------------- 1. operator, per-sequence truth
CASES = {
    "edges_4k": (16, 4096, [0] + _edges(4096) + [0, 0]),
    "edges_1M": (4, 1 << 20, _edges(1 << 20)),
    # offsets of every residue mod 4 (and mod 2) at the starts of sequences of each bucket, zero lengths between them
    "odd_offsets": (8, 4096, [3, 1, 0, 2, 1, 5, 1026, 7, 1023, 0, 2049, 2, 1, 3, 4095, 1]),
    "many_short": (8, 300, [1 + (7919 * i) % 300 for i in range(4096)]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_operator_against_per_sequence_truth(case):
    D, l_max, lengths = CASES[case]
    op, P = _make(D, l_max)
    u, cu = packed_input(lengths, D)
    dy = torch.randn(u.shape, generator=torch.Generator().manual_seed(5))
    _check_truth(_train(op, u, dy, torch.tensor(cu, dtype=torch.int32)), u, dy, cu, P, case)


def test_operator_64bit_offsets():
    """3 D total > 2^31: packed offsets of the high channels exceed int32.  dy is 0 except on the last sequence, so the
    parameter gradients are that sequence's alone and the truth stays small."""
    D = 256
    lengths = [1 << 20, 1 << 20, 700000, 1000]
    total = sum(lengths)
    assert 3 * D * total > 2 ** 31
    op, P = _make(D, 1 << 20)
    u, cu = packed_input(lengths, D)
    dy = torch.zeros(u.shape)
    dy[cu[-2]:] = torch.randn(lengths[-1], D, generator=torch.Generator().manual_seed(7))
    res = _train(op, u, dy, torch.tensor(cu, dtype=torch.int64, device=_dev()))
    _check_truth(res, u, dy, cu, P, "64-bit", only={3})


# ---------------------------------------------------------------------------------------------- 2. isolation, bit for bit
@pytest.mark.parametrize("fill", ["random", "nan", "inf"])
def test_sequence_bits_do_not_depend_on_neighbours_or_place(fill):
    """The target sequence's y and du keep their bits when its neighbours change contents (NaN and +-inf included) and
    order, and it moves in the pack; the buckets keep their sizes, so the same kernels run."""
    D = 16
    op, _ = _make(D, 4096)
    lengths = [5, 1030, 300, 2049, 77, 1]
    u, cu = packed_input(lengths, D)
    dy = torch.randn(u.shape, generator=torch.Generator().manual_seed(9))
    y0, du0, _ = _train(op, u, dy, torch.tensor(cu))
    tgt = 2
    a, b = cu[tgt], cu[tgt + 1]
    order = [3, 0, 5, 1, 2, 4]                                  # the target becomes the fifth sequence
    g = torch.Generator().manual_seed(11)
    parts, dparts = [], []
    for i in order:
        s, e = cu[i], cu[i + 1]
        if i == tgt:
            parts.append(u[s:e]); dparts.append(dy[s:e])
            continue
        x = torch.randn(e - s, D, generator=g) * 3
        if fill == "nan":
            x[::2] = float("nan")
        elif fill == "inf":
            x = torch.where(torch.rand(x.shape, generator=g) < 0.5, float("inf"), float("-inf"))
        parts.append(x); dparts.append(torch.randn(e - s, D, generator=g))
    u2, dy2 = torch.cat(parts), torch.cat(dparts)
    cu2 = [0]
    for i in order:
        cu2.append(cu2[-1] + lengths[i])
    y2, du2, _ = _train(op, u2, dy2, torch.tensor(cu2))
    a2 = cu2[order.index(tgt)]
    assert torch.equal(y2[a2:a2 + b - a], y0[a:b]), "the target's outputs changed with its neighbours"
    assert torch.equal(du2[a2:a2 + b - a], du0[a:b]), "the target's du changed with its neighbours"


def test_no_grad_gives_the_autograd_bits():
    D = 16
    op, _ = _make(D, 4096)
    u, cu = packed_input([3, 1500, 1024, 2, 4000], D)
    cut = torch.tensor(cu)
    y1, _, _ = _train(op, u, torch.ones(u.shape), cut)
    with torch.no_grad():
        y0 = op(u.to(_dev()), cu_seqlens=cut)
    assert torch.equal(y0, y1)
    y3 = op(u.to(_dev())[None], cu_seqlens=cut, max_seqlen=4000)      # (1, total, D) and max_seqlen
    assert y3.shape == (1,) + tuple(u.shape) and torch.equal(y3[0].detach(), y1)


# ---------------------------------------------------------------------------------------------- 3. Block and Backbone
@pytest.mark.parametrize("via", ["backbone", "block"])
def test_backbone_with_mlp_against_fp64_composition(via):
    """A two-layer Backbone with Mlp on (total, D) packed input, called with cu_seqlens (validated once) or layer by layer
    through Block(mixer_kwargs={"cu_seqlens", "max_seqlen"}), against the fp64 composition on each sequence alone."""
    H = _H()
    dev = _dev()
    D, n_layer, l_max = 32, 2, 4096
    lengths = [700, 1, 1025, 0, 3, 4096, 33]
    g = torch.Generator().manual_seed(3)
    torch.manual_seed(3)
    mixer = partial(H.HyenaOperator, l_max=l_max, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh"))
    m = H.Backbone(D, n_layer, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    _ln_randomize(m, g)
    m = m.to(dev)
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    x = torch.randn(cu[-1], D, generator=g)
    dy = torch.randn(cu[-1], D, generator=g)
    xg = x.to(dev).requires_grad_(True)
    cut = torch.tensor(cu, dtype=torch.int32, device=dev)
    if via == "backbone":
        y = m(xg, cu_seqlens=cut, max_seqlen=max(lengths))
    else:
        h, res = xg, None
        for layer in m.layers:
            h, res = layer(h, res, mixer_kwargs={"cu_seqlens": cut, "max_seqlen": max(lengths)})
        y, _ = H.Block._add_norm(h, res, m.ln_f)
    y.backward(dy.to(dev))
    ref, out = {}, {}
    for bits, dt in ((32, torch.float32), (64, torch.float64)):
        ref[bits] = _leaves(m, dev, dt)
        ys, dxs = [], []
        for a, b in zip(cu[:-1], cu[1:]):
            if b == a:
                continue
            xx = x[a:b][None].to(dev, dt).requires_grad_(True)
            yy = backbone_ref(xx, ref[bits], n_layer, dt)
            yy.backward(dy[a:b][None].to(dev, dt))
            ys.append(yy.detach()[0]); dxs.append(xx.grad[0])
        out[bits] = (torch.cat(ys), torch.cat(dxs))
    _act(y, out[32][0], out[64][0], f"packed backbone via {via} y")
    _act(xg.grad, out[32][1], out[64][1], f"packed backbone via {via} dx")
    _check_grads(m, ref, f"packed backbone via {via}")


# ---------------------------------------------------------------------------------------------- 4. launches
def test_one_launch_per_pass_per_bucket():
    """Forward + backward of 300 sequences in three buckets: every FFT pass and the short-filter backward launch once per
    bucket (one channel group), whatever the number of sequences."""
    H = _H()
    D = 8
    op, _ = _make(D, 4096)
    lengths = [1 + (37 * i) % 1024 for i in range(100)] + [1025 + i for i in range(100)] + [2049 + 3 * i for i in range(100)]
    u, cu = packed_input(lengths, D)
    cut = torch.tensor(cu)
    _train(op, u, torch.ones(u.shape), cut)                     # warm: workspaces, twiddles
    H._lib.profile_begin()
    _train(op, u, torch.ones(u.shape), cut)
    prof = H._lib.profile_end()
    n = {k: v[1] for k, v in prof.items()}
    nb = 3
    assert n["col_fwd<gate>"] == nb, n                  # forward only: the backward reuses the saved g spectrum
    assert n["col_fwd<dc>"] == nb and n["col_inv<conv_fwd>"] == nb and n["col_inv<bwd_dg>"] == nb, n
    assert n["col_inv<dk>"] == nb and n["short_conv_bwd"] == nb, n
    assert n["row_pass<conv_fwd>"] == nb and n["row_pass<conv_bwd>"] == nb, n
