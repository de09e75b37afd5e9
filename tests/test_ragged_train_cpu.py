"""Training on left-padded batches (``mask=``, hyena_b200_core_bwd_rows; DESIGN.md section 4.17) without a GPU: the guards
of the C entry point and the host validation of HyenaOperator, Block and Backbone, each firing before any device work;
the per-row d in_proj.bias formula; and self-checks that the per-row truth the GPU tests use rejects planted masking
bugs."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O

_lib = import_module("hyena_dna_b200._lib")

PTR = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


def test_abi_present_and_no_new_kinds():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    assert "hyena_b200_core_bwd_rows" in _lib.SIGNATURES and hasattr(L, "hyena_b200_core_bwd_rows")
    assert "hyena_b200_core_bwd_rows(" in header
    assert L.hyena_b200_abi_version() == 3 and L.hyena_b200_kind_count() == 33


def _core_bwd(dy=PTR, p=PTR, kspec=PTR, c=PTR, dk=PTR, ds=PTR, rs=PTR, ib=None, gs=None, dp=None, dib=None, B=2, D=8,
              Lq=1024):
    return _lib.lib().hyena_b200_core_bwd_rows(dy, p, ib, PTR, PTR, kspec, PTR, c, gs, dp, dk, PTR, PTR, PTR, dib, ds, rs,
                                               B, D, Lq, PTR, 1 << 30, None)


def test_core_bwd_rows_guards():
    n0 = _lib.launch_count()
    odd, odd8 = ctypes.c_void_p(258), ctypes.c_void_p(260)
    for kw, msg in [(dict(rs=None), "null pointer"), (dict(dy=None), "null pointer"), (dict(p=None), "null pointer"),
                    (dict(c=None), "null pointer"), (dict(dk=None), "null pointer"), (dict(ds=None), "null pointer"),
                    (dict(kspec=None), "null pointer"), (dict(B=0), "bad shape"), (dict(D=0), "bad shape"),
                    (dict(Lq=0), "bad shape"), (dict(Lq=(1 << 20) + 1), "exceeds the supported maximum"),
                    (dict(B=65536), "too large"), (dict(dy=odd), "misaligned"), (dict(p=odd), "misaligned"),
                    (dict(rs=odd), "misaligned"), (dict(ds=odd), "misaligned"), (dict(dp=odd), "misaligned"),
                    (dict(ib=odd), "misaligned"), (dict(dib=odd), "misaligned"), (dict(c=odd), "misaligned"),
                    (dict(kspec=odd8), "misaligned"), (dict(gs=odd8), "misaligned")]:
        assert _core_bwd(**kw) != 0 and msg in _err(), (kw, _err())
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- host validation
@pytest.fixture
def no_device(monkeypatch):
    """Every device entry point of the masked forward fails the test if reached."""
    H = _H()
    for name in ("core_forward", "core_backward", "proj_gemm", "proj_wgrad", "add_layer_norm", "filter_spectrum",
                 "filter_forward", "fftconv_forward"):
        monkeypatch.setattr(H.ops, name, lambda *a, _n=name, **k: pytest.fail(f"device work ({_n}) before validation"))
    return H


def _left(lengths, P):
    return torch.stack([torch.arange(P) >= P - n for n in lengths])


BAD_MASKS = [
    (torch.tensor([[0, 1, 1, 1, 1, 1, 1, 1], [0, 0, 1, 0, 1, 1, 1, 1], [1] * 8]), "row 1 is not left-padded"),
    (torch.tensor([[1] * 8, [1] * 8, [1, 1, 1, 1, 0, 0, 0, 0]]), "row 2 is not left-padded"),   # right-padded
    (torch.tensor([[1] * 8, [0] * 8, [1] * 8]), "row 1 is empty"),
    (torch.ones(3, 7, dtype=torch.bool), r"must be \(3, 8\)"),
    (torch.ones(2, 8, dtype=torch.bool), r"must be \(3, 8\)"),
    (torch.ones(3, 8, 1, dtype=torch.bool), r"must be \(3, 8\)"),
    (torch.ones(3, 8), "bool or integer"),
    (torch.ones(3, 8, dtype=torch.float64), "bool or integer"),
    (torch.full((3, 8), 2), "0 or 1"),
    ([[1] * 8] * 3, "bool or integer tensor"),
]


@pytest.mark.parametrize("mask,msg", BAD_MASKS)
@pytest.mark.parametrize("order", [2, 3])
def test_masks_are_validated_first(no_device, mask, msg, order):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5, order=order)
    u = torch.zeros(3, 8, 8, requires_grad=True)
    n0 = H.launch_count()
    with pytest.raises(H.HyenaB200Error, match=msg):
        op(u, mask=mask)
    with torch.no_grad(), pytest.raises(H.HyenaB200Error, match=msg):
        op(u, mask=mask)
    assert H.launch_count() == n0


def test_mask_combinations_and_operator_limits(no_device):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    u = torch.zeros(3, 8, 8)
    m = _left([8, 1, 5], 8)
    n0 = H.launch_count()
    with pytest.raises(H.HyenaB200Error, match="not both"):
        op(u, mask=m, lengths=[8, 1, 5])
    cache = H.DecodeCache(op, 3, 64, 64, torch.zeros(8 * 64 + 4), torch.zeros(8), torch.zeros(1, 3, 8, 64),
                          torch.zeros(3, 24, 2), torch.zeros(3, 24), torch.zeros(3, 8, 1))
    with pytest.raises(H.HyenaB200Error, match="DecodeCache"):
        op(u, mask=m, inference_params=cache)
    with pytest.raises(H.HyenaB200Error, match="l_max"):
        op(torch.zeros(3, 65, 8), mask=torch.ones(3, 65, dtype=torch.bool))
    with pytest.raises(H.HyenaB200Error, match=r"\(B, L, 8\)"):
        op(torch.zeros(3, 8, 7), mask=m)
    bidir = H.HyenaOperator(8, 64, emb_dim=5, bidirectional=True)
    with pytest.raises(H.HyenaB200Error, match="bidirectional"):
        bidir(u, mask=m)
    # a valid mask (bool, int, on the CPU) passes every host check: on the CPU the next thing that fails is the device
    for mm in (m, m.to(torch.int64), m.to(torch.uint8), m.to(torch.int32)):
        with pytest.raises(H.HyenaB200Error, match="CUDA"):
            op(u.requires_grad_(True), mask=mm)
    assert H.launch_count() == n0


def test_lengths_keeps_its_training_error(no_device):
    H = no_device
    op = H.HyenaOperator(8, 64, emb_dim=5)
    with pytest.raises(H.HyenaB200Error, match="pad them on the right") as e:
        op(torch.zeros(3, 8, 8), lengths=[8, 8, 8])
    assert "mask=" in str(e.value)


def test_block_and_backbone_validate_before_the_first_kernel(no_device):
    H = no_device
    mixer = partial(H.HyenaOperator, l_max=64, emb_dim=5)
    block = H.Block(8, mixer_cls=mixer, mlp_cls=partial(H.Mlp, hidden_features=16))
    bb = H.Backbone(8, 2, mixer, mlp_cls=partial(H.Mlp, hidden_features=16))
    u = torch.zeros(3, 8, 8, requires_grad=True)
    n0 = H.launch_count()
    for mask, msg in BAD_MASKS:
        with pytest.raises(H.HyenaB200Error, match=msg):
            block(u, mask=mask)
        with pytest.raises(H.HyenaB200Error, match=msg):
            bb(u, mask=mask)
    m = _left([8, 1, 5], 8)
    with pytest.raises(H.HyenaB200Error, match="not both"):
        block(u, mask=m, lengths=[8, 1, 5])
    with pytest.raises(H.HyenaB200Error, match="not both"):
        bb(u, mask=m, lengths=[8, 1, 5])
    cache = H.DecodeCache(block.mixer, 3, 64, 64, torch.zeros(8 * 64 + 4), torch.zeros(8), torch.zeros(1, 3, 8, 64),
                          torch.zeros(3, 24, 2), torch.zeros(3, 24), torch.zeros(3, 8, 1))
    with pytest.raises(H.HyenaB200Error, match="DecodeCache"):
        block(u, mask=m, mixer_kwargs={"inference_params": cache})
    with pytest.raises(H.HyenaB200Error, match="CUDA"):        # valid: the device check is next
        block(u, mask=m)
    assert H.launch_count() == n0


# ---------------------------------------------------------------------------------------------- d in_proj.bias per row
@pytest.mark.parametrize("lengths,L", [([12, 1, 2, 7], 12), ([1, 1], 5), ([2, 9, 3], 9), ([1], 1), ([2, 1], 2),
                                       ([15, 12, 0, 3], 12), ([9, -5, 2, 10], 9), ([2, 0], 1), ([3, -1], 2)])
def test_rows_in_bias_grad_matches_autograd(lengths, L):
    """d in_proj.bias = d/d bias of sum_t ds[t] * short(where(t >= s_b, p + bias, 0))[t] in fp64 autograd, against the
    per-row edge formula of ops.rows_in_bias_grad (ds zero at the pads, as core_bwd_rows leaves it).  A length > L is a
    start < 0, which masks nothing; a length <= 0 is a start >= L, which masks the whole row."""
    H = _H()
    g = torch.Generator().manual_seed(len(lengths) * 100 + L)
    B, C = len(lengths), 6
    starts = torch.tensor([L - n for n in lengths], dtype=torch.int32)
    keep = (torch.arange(L)[None, :] >= starts[:, None].long())[:, None, :]
    p = torch.randn(B, C, L, generator=g, dtype=torch.float64)
    w = torch.randn(C, 1, 3, generator=g, dtype=torch.float64)
    sb = torch.randn(C, generator=g, dtype=torch.float64)
    ds = torch.where(keep, torch.randn(B, C, L, generator=g, dtype=torch.float64), 0.0)
    bias = torch.randn(C, generator=g, dtype=torch.float64, requires_grad=True)
    x = torch.where(keep, p + bias[None, :, None], 0.0)
    s = F.conv1d(x, w, sb, padding=2, groups=C)[..., :L]
    (s * ds).sum().backward()
    got = H.ops.rows_in_bias_grad(ds, w.reshape(C, 3), ds.sum((0, 2)), starts)
    assert torch.allclose(got, bias.grad, rtol=1e-12, atol=1e-12), (got - bias.grad).abs().max()


# ---------------------------------------------------------------------------------------------- the per-row truth
def row_truth(u, dy, lengths, P, dtype):
    """Truth of a left-padded batch: the oracle (O.operator_fwd_bwd) on each row's UNPADDED tokens in ``dtype`` -> (list
    of per-row y, list of per-row du, parameter gradients summed over the rows)."""
    L = u.shape[1]
    Q = O.to_dtype(P, dtype)
    ys, dus, sums = [], [], {}
    for b, n in enumerate(lengths):
        y, du, g = O.operator_fwd_bwd(u[b:b + 1, L - n:].to(dtype), Q, dy[b:b + 1, L - n:].to(dtype))
        ys.append(y)
        dus.append(du)
        for k, v in g.items():
            sums[k] = sums.get(k, 0) + v
    return ys, dus, sums


def masked_model(u, dy, lengths, P, bug=None):
    """The masked operator on the padded batch in fp64 autograd, masked where the library masks (u at the pads, the short
    filter's input, g and y_pre) -> (y, du, parameter gradients).  ``bug`` plants one masking error that changes only
    gradients (the forward values are unchanged: x - x.detach() adds an exact 0):
      "leak": the transposed short filter carries ds into s_b - 1 (u not zeroed at the pads, dp not masked there);
      "bias": d in_proj.bias summed over the pads as well;
      "tap":  d short_filter.weight read from unmasked pad samples."""
    B, L, D = u.shape
    Q = {k: v.detach().clone().double().requires_grad_(k not in ("filter_fn.pos_emb.z", "filter_fn.pos_emb.t",
                                                                  "filter_fn.modulation.deltas")) for k, v in P.items()}
    u = u.detach().clone().double().requires_grad_(True)
    s = torch.tensor([L - n for n in lengths])
    t = torch.arange(L)
    keep = (t[None, :] >= s[:, None])[:, None, :]                               # (B, 1, L)
    uin = u if bug == "leak" else torch.where(keep.transpose(1, 2), u, 0.0)
    W, ib = Q["in_proj.weight"], Q["in_proj.bias"]
    order = W.shape[0] // D - 1
    p_raw = F.linear(uin, W, ib).transpose(1, 2)
    x_in = torch.where(keep, p_raw, 0.0)
    if bug == "leak":
        x_in = x_in + (p_raw - p_raw.detach()) * (t[None, None, :] == s[:, None, None] - 1)
    if bug == "bias":
        x_in = x_in + (ib - ib.detach())[None, :, None] * ~keep
    sw, sb = Q["short_filter.weight"], Q["short_filter.bias"]
    if bug == "tap":
        uc = O.short_filter(x_in, sw.detach(), sb, L)
        tap = O.short_filter(p_raw.detach(), sw, None, L)
        uc = uc + (tap - tap.detach())
    else:
        uc = O.short_filter(x_in, sw, sb, L)
    *x, v = uc.split(D, dim=1)
    k = O.hyena_filter(L, Q)[0].transpose(0, 1).reshape(D, order - 1, L)
    fb = Q["filter_fn.bias"].reshape(D, order - 1)
    for o, x_i in enumerate(reversed(x[1:])):
        g = torch.where(keep, v * x_i, 0.0)
        v = O.fftconv_ref(g, k[:, o], fb[:, o])
    y_pre = torch.where(keep, v * x[0], 0.0).transpose(1, 2)
    y = F.linear(y_pre, Q["out_proj.weight"], Q["out_proj.bias"])
    y.backward(dy.double())
    return y.detach(), u.grad.detach(), {k: q.grad.detach() for k, q in Q.items() if q.grad is not None}


def _agree(a, b, tol=1e-9):
    return a.shape == b.shape and bool(((a - b).abs() <= tol * (1.0 + b.abs().max())).all())


def _case(order=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    D, L, lmax = 4, 23, 32
    P = O.init_params(D, lmax, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.3)
    P["in_proj.bias"] = 0.3 * torch.randn(P["in_proj.bias"].shape, generator=g)
    P["short_filter.bias"] = 0.3 * torch.randn(P["short_filter.bias"].shape, generator=g)
    lengths = [23, 1, 2, 10]
    u = torch.randn(len(lengths), L, D, generator=g, dtype=torch.float64)
    dy = torch.randn(len(lengths), L, D, generator=g, dtype=torch.float64)
    for b, n in enumerate(lengths):
        u[b, :L - n] = 3.0 * torch.randn(L - n, D, generator=g, dtype=torch.float64)       # pads: not zero
        dy[b, :L - n] = 0.0                                                                  # the loss sees real positions
    return P, u, dy, lengths


def _compare(model, truth, lengths, L):
    y, du, grads = model
    ys, dus, sums = truth
    ok = True
    for b, n in enumerate(lengths):
        ok &= _agree(y[b:b + 1, L - n:], ys[b]) and _agree(du[b:b + 1, L - n:], dus[b])
        ok &= bool((du[b, :L - n] == 0).all())
    for k in sums:
        ok &= _agree(grads[k].reshape(sums[k].shape), sums[k])
    return ok


@pytest.mark.parametrize("order", [2, 3])
def test_masked_model_matches_the_per_row_truth(order):
    P, u, dy, lengths = _case(order)
    truth = row_truth(u, dy, lengths, P, torch.float64)
    assert len(truth[2]) == 15 if order == 2 else len(truth[2]) >= 15
    assert _compare(masked_model(u, dy, lengths, P), truth, lengths, u.shape[1])


@pytest.mark.parametrize("bug", ["leak", "bias", "tap"])
@pytest.mark.parametrize("order", [2, 3])
def test_per_row_truth_rejects_planted_bugs(order, bug):
    P, u, dy, lengths = _case(order)
    truth = row_truth(u, dy, lengths, P, torch.float64)
    model = masked_model(u, dy, lengths, P, bug=bug)
    for b, n in enumerate(lengths):                                   # the forward values are the correct ones
        assert _agree(model[0][b:b + 1, u.shape[1] - n:], truth[0][b])
    assert not _compare(model, truth, lengths, u.shape[1]), f"planted bug {bug!r} went unnoticed"
