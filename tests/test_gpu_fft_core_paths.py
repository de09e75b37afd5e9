"""The order-2 FFT core's dispatch paths against fp64.

The host code of the long convolution (csrc/api.cu, csrc/k_row.cu) picks a kernel, or a code path inside one, from the
shape and the addresses of its inputs.  Each test below drives one family of those decisions on purpose and compares
every output with an fp64 restatement of the same operation (``core_ref``), through tests/parity_util.check:

| decision                                                   | selected by                       | test                                   |
|------------------------------------------------------------|-----------------------------------|----------------------------------------|
| transform template LOGM1 = 0..10, TWO / G-column geometry  | L                                 | test_fused_core_sweep, test_unfused_core |
| staged row pass vs row_pass_kernel<ROW_CONV_FWD>           | L (LOGM1 >= 2), kspec alignment   | test_fused_core_sweep, test_operand_addresses[kspec8] |
| batch-1 backward: staged / unstaged BWD1 / ROW_CONV_BWD    | B, saved gspec, alignment         | test_fused_core_sweep, test_operand_addresses[kspec8], test_spectrum_recompute |
| cp.async column staging (a.stage) vs direct loads          | L mod 4, 16-byte rows             | test_fused_core_sweep, test_operand_addresses[p8] |
| float2 accesses (a.vec)                                    | L parity, 8-byte rows             | test_fused_core_sweep, test_operand_addresses[p4] |
| channel groups (carve, c0 > 0, ragged last group)          | workspace size, D > 65535 / B     | test_channel_groups_bitwise, test_operator_batch_300_groups, test_core_full_length_groups |
| un-fused core: core_bwd with dp, short_conv_bwd            | L > l_max, proj mode              | test_unfused_core, test_operator_longer_than_l_max, test_operator_unfused_routes |
| spectrum recompute (gspec == NULL)                         | HYENA_B200_SAVE_SPECTRUM=0        | test_spectrum_recompute                |

Activations are held to 1e-3 rel with the absolute term scaled by max|ref|, parameter gradients with ``param_grad=True``;
the fp32 twin of the reference (``ref32``) and its fp64 truth (``ref64``) are both passed, so the S8(c) hatch can apply
and is book-kept.  The tests marked ``gpu`` need an H100; the reference self-checks at the top run on the CPU.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------ fp64 reference of the core
def core_ref(x, ib, sw, sb, k, fb, dy, dtype=torch.float64, W=None, conv=O.fftconv_ref):
    """Order-2 Hyena core with the filter k given directly (hyena.py:391-439 without the filter MLP and out_proj).

    x is u (B, L, D) when W (3D, D) is given (in_proj without its bias), else p (B, 3D, L), the in_proj output without
    its bias.  ib (3D,) in_proj bias, sw (3D, 3) short-filter taps, sb (3D,), k (D, L), fb (D,), dy (B, D, L).
    Returns y_pre = c * x0 (B, D, L) and c = fftconv(v * x1, k, fb), with the gradients of every input under dy:
    dx (du or dp), dW, dib, dsw, dsb, dk, dfb, and ds, the gradient of the short-filter output (B, 3D, L)."""
    leaves = [t.detach().to(dtype).clone().requires_grad_(True) for t in (x, ib, sw, sb, k, fb)]
    x_, ib_, sw_, sb_, k_, fb_ = leaves
    W_ = W.detach().to(dtype).clone().requires_grad_(True) if W is not None else None
    p = F.linear(x_, W_).transpose(1, 2) if W_ is not None else x_
    C3, L = p.shape[1], p.shape[2]
    D = C3 // 3
    uc = O.short_filter(p + ib_[None, :, None], sw_.reshape(C3, 1, 3), sb_, L)
    uc.retain_grad()
    x0, x1, v = uc.split(D, dim=1)
    c = conv(v * x1, k_, fb_)
    y = c * x0
    y.backward(dy.to(dtype))
    out = dict(y=y.detach(), c=c.detach(), dx=x_.grad, dib=ib_.grad, dsw=sw_.grad, dsb=sb_.grad, dk=k_.grad,
               dfb=fb_.grad, ds=uc.grad)
    if W_ is not None:
        out["dW"] = W_.grad
    return out


def core_refs(*args, **kw):
    """(fp32 reference, fp64 truth) of core_ref on the host."""
    return core_ref(*args, dtype=torch.float32, **kw), core_ref(*args, dtype=torch.float64, **kw)


def decaying_filter(D, L, g):
    """A random causal filter with unit-ish gain (like a trained Hyena filter), so outputs stay near unit scale."""
    return torch.randn(D, L, generator=g) * torch.exp(-torch.arange(L) / (0.05 * L + 1))[None] / math.sqrt(0.05 * L + 1)


def core_inputs(B, D, L, seed, with_u=False):
    """Seeded host inputs of one core call."""
    g = torch.Generator().manual_seed(seed)
    t = dict(p=torch.randn(B, 3 * D, L, generator=g), ib=torch.randn(3 * D, generator=g) * 0.5,
             sw=(torch.rand(3 * D, 3, generator=g) * 2 - 1) / math.sqrt(3), sb=(torch.rand(3 * D, generator=g) * 2 - 1) / math.sqrt(3),
             k=decaying_filter(D, L, g), fb=torch.randn(D, generator=g), dy=torch.randn(B, D, L, generator=g))
    if with_u:
        t["u"] = torch.randn(B, L, D, generator=g)
        t["W"] = torch.randn(3 * D, D, generator=g) / math.sqrt(D)
    return t


def _act(got, r32, r64, what):
    """Activation against fp64: absolute term scaled by max|ref| (tests/test_gpu_parity.py::_close)."""
    s = max(1.0, float(r64.detach().abs().max()))
    return PU.check(got, r32, what + (f" [abs term x{s:.3g}]" if s > 1.0 else ""), ref64=r64, atol=PU.ATOL * s)


def _par(got, r32, r64, what):
    return PU.check(got, r32, what, ref64=r64, param_grad=True)


# ------------------------------------------------------------------------------------------ CPU self-checks of the reference
@pytest.mark.parametrize("B,L,D", [(2, 37, 4), (1, 130, 6)])
def test_core_ref_matches_operator_oracle_and_direct_convolution(B, L, D):
    """core_ref is the oracle operator's core: same y_pre as hyena_operator's intermediate, and the same outputs and
    gradients when its FFT convolution is replaced by the O(L^2) time-domain sum."""
    g = torch.Generator().manual_seed(L)
    P = O.to_dtype(O.init_params(D, L, emb_dim=5, w=1.0, generator=g), torch.float64)
    u = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    _, inter = O.hyena_operator(u, P, return_intermediates=True)
    dy = torch.randn(B, D, L, generator=g, dtype=torch.float64)
    args = (u, P["in_proj.bias"], P["short_filter.weight"].reshape(3 * D, 3), P["short_filter.bias"], inter["k"],
            P["filter_fn.bias"], dy)
    r = core_ref(*args, W=P["in_proj.weight"])
    torch.testing.assert_close(r["y"], inter["y_pre"].transpose(1, 2), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["c"], inter["c"], rtol=1e-12, atol=1e-12)
    d = core_ref(*args, W=P["in_proj.weight"], conv=O.fftconv_direct)
    for name in ("y", "c", "dx", "dW", "dib", "dsw", "dsb", "dk", "dfb", "ds"):
        torch.testing.assert_close(r[name], d[name], rtol=1e-10, atol=1e-10, msg=name)


@pytest.mark.parametrize("L", [300, 4097])
def test_parity_bar_rejects_perturbed_cores(L):
    """The tolerance can tell a correct core from the bugs a kernel would make: a filter shifted by one tap, a dropped
    filter bias, two short-filter taps swapped in one channel, a zeroed last position.  Each perturbed fp64 output must
    be rejected against the unperturbed fp32 / fp64 pair that a correct output passes."""
    B, D = 2, 4
    t = core_inputs(B, D, L, seed=L)
    args = [t["p"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"]]
    r32, r64 = core_refs(*args)
    n0 = len(PU._records)
    try:
        _act(r64["y"].float(), r32["y"], r64["y"], "unperturbed")
        k_shift = F.pad(t["k"], (1, 0))[:, :L]
        sw_swap = t["sw"].clone()
        sw_swap[1, [0, 1]] = sw_swap[1, [1, 0]]
        perturbed = {"k shifted one tap": core_ref(*args[:4], k_shift, *args[5:])["y"],
                     "filter bias dropped": core_ref(*args[:5], torch.zeros_like(t["fb"]), args[6])["y"],
                     "short-filter taps swapped": core_ref(*args[:2], sw_swap, *args[3:])["y"]}
        last = r64["y"].clone()
        last[..., -1] = 0
        perturbed["last position zeroed"] = last
        for what, y in perturbed.items():
            with pytest.raises(AssertionError):
                _act(y, r32["y"], r64["y"], what)
    finally:
        del PU._records[n0:]            # self-checks of the bar, not parity records


# ------------------------------------------------------------------------------------------ device helpers
def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _leaf(t, dev):
    return t.to(dev).requires_grad_(True)


def _check_core_grads(got, r32, r64, tag, names=("dib", "dsw", "dsb", "dk", "dfb")):
    for n in names:
        _par(got[n], r32[n], r64[n], f"{tag} grad {n}")


# ------------------------------------------------------------------------------------------ 2. transform size x residue sweep
SWEEP_L = [1, 2, 3, 5, 255, 1024, 1025, 2046, 2051, 4096, 4097, 8190, 12289, 16384, 16385, 32766, 32768, 40000, 65535,
           100001, 131072, 160002, 262144, 300000, 524287, 524289, 1048574, 1048576]


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", SWEEP_L)
def test_fused_core_sweep(L, B):
    """HyenaInCoreFn (in_proj GEMM + fused core + ds-fed projection backward) at every transform size, both sides of each
    power of two, every L mod 4 on the TWO sizes and the tiny edges of the 3-tap filter."""
    H = _H()
    dev = _dev()
    D = 4
    t = core_inputs(B, D, L, seed=7 * L + B, with_u=True)
    r32, r64 = core_refs(t["u"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"], W=t["W"])
    u, W, ib, sw, sb, k, fb = (_leaf(t[n], dev) for n in ("u", "W", "ib", "sw", "sb", "k", "fb"))
    y = H.ops.HyenaInCoreFn.apply(u, W, ib, sw.reshape(3 * D, 1, 3), sb, k, fb)
    y.backward(t["dy"].to(dev))
    tag = f"fused core B={B} L={L}"
    _act(y, r32["y"], r64["y"], f"{tag} y_pre")
    _act(u.grad, r32["dx"], r64["dx"], f"{tag} du")
    got = dict(dW=W.grad, dib=ib.grad, dsw=sw.grad, dsb=sb.grad, dk=k.grad, dfb=fb.grad)
    _check_core_grads(got, r32, r64, tag, ("dW", "dib", "dsw", "dsb", "dk", "dfb"))


UNFUSED_L = [1000, 2046, 4096, 8190, 12289, 32766, 40000, 100001, 160002, 300000, 524289]    # LOGM1 = 0 .. 10


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", UNFUSED_L)
def test_unfused_core(L, B):
    """HyenaCoreFn: core_bwd writes dp through short_conv_bwd_kernel (the path of L > l_max and the non-wgmma modes)."""
    H = _H()
    dev = _dev()
    D = 4
    t = core_inputs(B, D, L, seed=11 * L + B)
    r32, r64 = core_refs(t["p"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"])
    p, ib, sw, sb, k, fb = (_leaf(t[n], dev) for n in ("p", "ib", "sw", "sb", "k", "fb"))
    y = H.ops.HyenaCoreFn.apply(p, ib, sw.reshape(3 * D, 1, 3), sb, k, fb)
    y.backward(t["dy"].to(dev))
    tag = f"unfused core B={B} L={L}"
    _act(y, r32["y"], r64["y"], f"{tag} y_pre")
    _act(p.grad, r32["dx"], r64["dx"], f"{tag} dp")
    _check_core_grads(dict(dib=ib.grad, dsw=sw.grad, dsb=sb.grad, dk=k.grad, dfb=fb.grad), r32, r64, tag)


# ------------------------------------------------------------------------------------------ 3. operand addresses
def _at_offset(t, nbytes):
    """A contiguous copy of t whose data starts nbytes past a fresh (256-byte aligned) allocation."""
    esz = t.element_size()
    assert nbytes % esz == 0
    off = nbytes // esz
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 == nbytes % 16
    return v


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", [4096, 40000, 1 << 20])
@pytest.mark.parametrize("where", ["p4", "p8", "kspec8"])
def test_operand_addresses(where, L, B):
    """core_forward / core_backward with operands at a storage offset.  p4: p, dy_pre and c_saved 4 bytes off (no float2
    accesses, vec = 0); p8: 8 bytes off (vec = 1, no cp.async column staging); kspec8: the filter spectrum one complex64
    element off, which selects the unstaged row_pass_kernel<ROW_CONV_FWD> and, at B = 1, <ROW_CONV_BWD1>."""
    H = _H()
    dev = _dev()
    D = 4
    t = core_inputs(B, D, L, seed=13 * L + B)
    r32, r64 = core_refs(t["p"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"])
    ib, sw, sb, k, fb = (t[n].to(dev) for n in ("ib", "sw", "sb", "k", "fb"))
    p, dy = t["p"].to(dev), t["dy"].to(dev)
    kspec = H.ops.filter_spectrum(k)
    if where == "kspec8":
        kspec = _at_offset(kspec, 8)
    else:
        off = 4 if where == "p4" else 8
        p, dy = _at_offset(p, off), _at_offset(dy, off)
    y, c, gs = H.ops.core_forward(p, ib, sw, sb, kspec, fb, True)
    if where != "kspec8":
        c = _at_offset(c, 4 if where == "p4" else 8)
    dp, dk, dsw, dsb, dfb, dib = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs)
    tag = f"addresses {where} B={B} L={L}"
    _act(y, r32["y"], r64["y"], f"{tag} y_pre")
    _act(c, r32["c"], r64["c"], f"{tag} c")
    _act(dp, r32["dx"], r64["dx"], f"{tag} dp")
    _check_core_grads(dict(dib=dib, dsw=dsw, dsb=dsb, dk=dk, dfb=dfb), r32, r64, tag)


# ------------------------------------------------------------------------------------------ 4. channel groups
def _exact_workspace(H, G):
    """A stand-in for ops.workspace that hands the library room for exactly G channels per group."""
    def ws(B, D, L, backward, device):
        n = int(H._lib.lib().hyena_b200_workspace_min_bytes(B, D, L, int(backward))) * G
        return torch.empty(n, dtype=torch.uint8, device=device)
    return ws


def _grouped_run(H, t, dev):
    ib, sw, sb, k, fb, p, dy = (t[n].to(dev) for n in ("ib", "sw", "sb", "k", "fb", "p", "dy"))
    uf, dout, Dv = t["uf"].to(dev), t["dout"].to(dev), t["Dv"].to(dev)
    o = {}
    o["kspec"] = H.ops.filter_spectrum(k)
    o["y"], o["c"], o["gspec"] = H.ops.core_forward(p, ib, sw, sb, o["kspec"], fb, True)
    o["dp"], o["dk"], o["dsw"], o["dsb"], o["dfb"], o["dib"] = H.ops.core_backward(dy, p, ib, sw, sb, o["kspec"], fb,
                                                                                   o["c"], o["gspec"])
    o["ds"] = H.ops.core_backward(dy, p, ib, sw, sb, o["kspec"], fb, o["c"], o["gspec"], return_ds=True)[0]
    o["fout"] = H.ops.fftconv_forward(uf, o["kspec"], Dv)
    o["fdu"], o["fdk"], o["fdD"] = H.ops.fftconv_backward(dout, uf, o["kspec"], Dv)
    torch.cuda.synchronize()
    return o


PER_ROW = ("kspec", "y", "c", "gspec", "dp", "ds", "dk", "fout", "fdu", "fdk")


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", [1000, 40000])
def test_channel_groups_bitwise(monkeypatch, L, B):
    """filter_spectrum, core fwd/bwd and fftconv fwd/bwd with the workspace cut to G = 1 and G = 3 channels per group
    (D = 8: eight groups, or 3 + 3 + 2): per-row outputs bit-identical to the one-group run, the atomically reduced
    sums within the fp64 tolerance, and one launch per group of each column pass."""
    H = _H()
    dev = _dev()
    D = 8
    t = core_inputs(B, D, L, seed=17 * L + B)
    g = torch.Generator().manual_seed(L + 5)
    t.update(uf=torch.randn(B, D, L, generator=g), dout=torch.randn(B, D, L, generator=g), Dv=torch.randn(D, generator=g))
    H._lib.profile_begin()
    base = _grouped_run(H, t, dev)
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 1 and prof["col_fwd<filter>"][1] == 1, prof
    r32, r64 = core_refs(t["p"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"])
    tag = f"groups B={B} L={L}"
    _act(base["y"], r32["y"], r64["y"], f"{tag} y_pre")
    _act(base["dp"], r32["dx"], r64["dx"], f"{tag} dp")
    _act(base["ds"], r32["ds"], r64["ds"], f"{tag} ds")
    fr = {}
    for dt in (torch.float32, torch.float64):
        uf, kk, Dv = (x.to(dt).clone().requires_grad_(True) for x in (t["uf"], t["k"], t["Dv"]))
        out = O.fftconv_ref(uf, kk, Dv)
        out.backward(t["dout"].to(dt))
        fr[dt] = dict(fout=out.detach(), fdu=uf.grad, fdk=kk.grad, fdD=Dv.grad)
    _act(base["fout"], fr[torch.float32]["fout"], fr[torch.float64]["fout"], f"{tag} fftconv out")
    _act(base["fdu"], fr[torch.float32]["fdu"], fr[torch.float64]["fdu"], f"{tag} fftconv du")
    for G in (1, 3):
        monkeypatch.setattr(H.ops, "workspace", _exact_workspace(H, G))
        H._lib.profile_begin()
        got = _grouped_run(H, t, dev)
        prof = H._lib.profile_end()
        ng = -(-D // G)
        assert prof["col_fwd<filter>"][1] == ng and prof["col_fwd<gate>"][1] == ng, prof
        assert prof["col_fwd<dc>"][1] == 2 * ng and prof["col_fwd<plain>"][1] == 3 * ng, prof
        for n in PER_ROW:
            assert torch.equal(got[n], base[n]), f"{tag} G={G}: {n} differs from the one-group run"
        _check_core_grads(got, r32, r64, f"{tag} G={G}", ("dib", "dsw", "dsb", "dfb"))
        _par(got["fdD"], fr[torch.float32]["fdD"], fr[torch.float64]["fdD"], f"{tag} G={G} fftconv grad dD")


def _operator(H, P, D, l_max, dev):
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = H.HyenaOperator(D, l_max, order=2, filter_order=64, emb_dim=5, w=1.0, lr_pos_emb=0.0)
    op.load_state_dict(sd, strict=True)
    return op.to(dev)


def _check_operator(H, op, u, dy, P, tag, dev, l_cut=None):
    """HyenaOperator fwd + bwd against the oracle operator (fp32 and fp64) on u[:, :l_cut]."""
    ug = u.to(dev).requires_grad_(True)
    y = op(ug)
    y.backward(dy.to(dev))
    lc = l_cut or u.shape[1]
    y32, du32, g32 = O.operator_fwd_bwd(u[:, :lc], P, dy)
    y64, du64, g64 = O.operator_fwd_bwd(u[:, :lc].double(), O.to_dtype(P, torch.float64), dy.double())
    assert tuple(y.shape) == tuple(y64.shape)
    _act(y, y32, y64, f"{tag} y")
    _act(ug.grad[:, :lc], du32, du64, f"{tag} du")
    got = dict(op.named_parameters())
    for name in g64:
        _par(got[name].grad, g32[name], g64[name], f"{tag} grad {name}")
    return ug.grad


@gpu
def test_operator_batch_300_groups():
    """B = 300 caps a launch at 65535 / 300 = 218 channels: D = 256 runs as 218 + 38 with the default workspace."""
    H = _H()
    dev = _dev()
    B, L, D = 300, 64, 256
    g = torch.Generator().manual_seed(300)
    P = O.init_params(D, L, emb_dim=5, w=1.0, generator=g)
    u = torch.randn(B, L, D, generator=g)
    dy = torch.randn(B, L, D, generator=g)
    op = _operator(H, P, D, L, dev)
    with torch.no_grad():
        H._lib.profile_begin()
        op(u.to(dev))
        prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 2, prof
    _check_operator(H, op, u, dy, P, "B=300 groups", dev)


@gpu
def test_core_full_length_groups():
    """B = 3, L = 2^20, D = 96 with the default workspace: 85 + 11 channels.  The core does not mix channels, so the
    channels on both sides of the boundary are checked against an fp64 run of those channels alone."""
    H = _H()
    dev = _dev()
    B, L, D = 3, 1 << 20, 96
    g = torch.Generator(device=dev).manual_seed(96)
    p = torch.randn(B, 3 * D, L, generator=g, device=dev)
    ib = torch.randn(3 * D, generator=g, device=dev) * 0.5
    sw = (torch.rand(3 * D, 3, generator=g, device=dev) * 2 - 1) / math.sqrt(3)
    sb = (torch.rand(3 * D, generator=g, device=dev) * 2 - 1) / math.sqrt(3)
    k = (torch.randn(D, L, generator=g, device=dev) * torch.exp(-torch.arange(L, device=dev) / (0.05 * L + 1))[None]
         / math.sqrt(0.05 * L + 1))
    fb = torch.randn(D, generator=g, device=dev)
    dy = torch.randn(B, D, L, generator=g, device=dev)
    kspec = H.ops.filter_spectrum(k)
    H._lib.profile_begin()
    y, c, gs = H.ops.core_forward(p, ib, sw, sb, kspec, fb, True)
    dp, dk, dsw, dsb, dfb, dib = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs)
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 2 and prof["col_fwd<dc>"][1] == 2, prof
    del c, gs
    ch = torch.tensor([0, 84, 85, 95])
    rows = torch.cat([ch, ch + D, ch + 2 * D])
    sub = lambda t, idx, dim: t.index_select(dim, idx.to(t.device)).cpu()
    r32, r64 = core_refs(sub(p, rows, 1), sub(ib, rows, 0), sub(sw, rows, 0), sub(sb, rows, 0), sub(k, ch, 0),
                         sub(fb, ch, 0), sub(dy, ch, 1))
    tag = "core groups 85+11 L=2^20"
    _act(sub(y, ch, 1), r32["y"], r64["y"], f"{tag} y_pre")
    _act(sub(dp, rows, 1), r32["dx"], r64["dx"], f"{tag} dp")
    got = dict(dib=sub(dib, rows, 0), dsw=sub(dsw, rows, 0), dsb=sub(dsb, rows, 0), dk=sub(dk, ch, 0), dfb=sub(dfb, ch, 0))
    _check_core_grads(got, r32, r64, tag)


# ------------------------------------------------------------------------------------------ 5. L > l_max, un-fused routes
@gpu
@pytest.mark.parametrize("l_max,L", [(1000, 1037), (20000, 20011)])
def test_operator_longer_than_l_max(l_max, L):
    """An input longer than l_max: the filter is l_max long, the output covers the first l_max positions (as the
    reference's), and the positions past it get a zero gradient."""
    H = _H()
    dev = _dev()
    B, D = 2, 8
    g = torch.Generator().manual_seed(L)
    P = O.init_params(D, l_max, emb_dim=5, w=1.0, generator=g)
    u = torch.randn(B, L, D, generator=g)
    dy = torch.randn(B, l_max, D, generator=g)
    op = _operator(H, P, D, l_max, dev)
    du = _check_operator(H, op, u, dy, P, f"L={L} > l_max={l_max}", dev, l_cut=l_max)
    assert tuple(du.shape) == (B, L, D)
    assert bool((du[:, l_max:] == 0).all())


@gpu
@pytest.mark.parametrize("route", ["proj_lt"])
def test_operator_unfused_routes(monkeypatch, route):
    """L == l_max through HyenaCoreFn and a separate short_conv_bwd pass, with the library projection GEMMs."""
    H = _H()
    dev = _dev()
    monkeypatch.setattr(H.ops, "_proj_mode", "lt" if H.ops.gemm_mode() == "bf16x9" else "torch")
    B, L, D = 2, 2999, 8
    g = torch.Generator().manual_seed(2999)
    P = O.init_params(D, L, emb_dim=5, w=1.0, generator=g)
    u = torch.randn(B, L, D, generator=g)
    dy = torch.randn(B, L, D, generator=g)
    op = _operator(H, P, D, L, dev)
    H._lib.profile_begin()
    _check_operator(H, op, u, dy, P, f"route {route}", dev)
    prof = H._lib.profile_end()
    assert "short_conv_bwd" in prof, prof


# ------------------------------------------------------------------------------------------ 6. spectrum recompute
@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", [1000, 4096, 40000, 1 << 20])
def test_spectrum_recompute(monkeypatch, L, B):
    """HYENA_B200_SAVE_SPECTRUM=0: the forward keeps no gate spectrum; the backward recomputes it (one more col_fwd<gate>)
    and, at B = 1, runs the batch-loop ROW_CONV_BWD instead of the batch-1 kernels."""
    monkeypatch.setenv("HYENA_B200_SAVE_SPECTRUM", "0")
    H = _H()
    dev = _dev()
    D = 4
    t = core_inputs(B, D, L, seed=19 * L + B, with_u=True)
    r32, r64 = core_refs(t["u"], t["ib"], t["sw"], t["sb"], t["k"], t["fb"], t["dy"], W=t["W"])
    u, W, ib, sw, sb, k, fb = (_leaf(t[n], dev) for n in ("u", "W", "ib", "sw", "sb", "k", "fb"))
    y = H.ops.HyenaInCoreFn.apply(u, W, ib, sw.reshape(3 * D, 1, 3), sb, k, fb)
    H._lib.profile_begin()
    y.backward(t["dy"].to(dev))
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 1, prof
    tag = f"recompute B={B} L={L}"
    _act(y, r32["y"], r64["y"], f"{tag} y_pre")
    _act(u.grad, r32["dx"], r64["dx"], f"{tag} du")
    got = dict(dW=W.grad, dib=ib.grad, dsw=sw.grad, dsb=sb.grad, dk=k.grad, dfb=fb.grad)
    _check_core_grads(got, r32, r64, tag, ("dW", "dib", "dsw", "dsb", "dk", "dfb"))

