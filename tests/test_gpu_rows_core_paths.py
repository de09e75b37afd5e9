"""The order-2 FFT core on left-padded rows against fp64: the masked modes at every transform size.

``ops.core_forward`` / ``ops.core_backward`` with ``row_start`` run COL_GATE_ROWS and INV_CONV_FWD_ROWS forward,
COL_DC_ROWS, INV_BWD_DG_ROWS (and COL_GATE_ROWS without a saved g spectrum) backward, and short_conv_bwd_rows_kernel
when dp is requested; ``return_ds=True`` leaves d in_proj.bias to ``ops.rows_in_bias_grad``.  Each mode is compiled once
per transform template LOGM1 = 0..10 (DESIGN.md section 4.17).  Every test below compares with ``rows_core_ref``: the
fp64 core (tests/test_gpu_fft_core_paths.core_ref) on each row's slice [s_b, L) alone, zero-extended at the pads, with
the parameter gradients summed over the rows.  The pads of p and dy_pre hold large values, never zeros, so a mask that
is missing shows.  Row starts are placed where a 3-tap window straddling them is hard to mask (``row_starts``).

| decision                                                  | selected by                     | test                             |
|-----------------------------------------------------------|---------------------------------|----------------------------------|
| transform template LOGM1 = 0..10, TWO / G-column geometry | L                               | test_rows_core_sweep             |
| starts on tile edges, their halo, 2048-sample column rows, | row_start                       | test_rows_core_sweep (row_starts) |
| staged-epilogue batches, short_conv_bwd spans              |                                 |                                  |
| cp.async staging / float2 (vec) / scalar accesses          | L mod 4, operand addresses      | test_rows_core_sweep, test_rows_operand_addresses, test_rows_register_path |
| short_conv_bwd_rows_kernel (dp) / rows_in_bias_grad (ds)   | return_ds                       | every GPU test                   |
| fused route: in_proj GEMM + core + ds-fed projections      | HyenaInCoreFn                   | test_rows_fused_route            |
| batch-1 backward: staged / unstaged ROW_CONV_BWD1          | B = 1, kspec alignment          | test_rows_batch_one              |
| spectrum recompute (COL_GATE_ROWS in the backward)         | HYENA_B200_SAVE_SPECTRUM=0      | test_rows_spectrum_recompute     |
| channel groups (c0 > 0, ragged last group)                 | workspace size                  | test_rows_channel_groups         |
| pad contents: zeros, random, NaN, +-inf                    | the caller's pads               | test_rows_pad_contents           |
| starts < 0 (mask nothing) and >= L (mask the whole row)    | row_start                       | test_rows_out_of_range_starts    |

Activations are held to 1e-3 rel with the absolute term scaled by max|ref|, parameter gradients with ``param_grad=True``,
both against the fp32 twin of the reference and its fp64 truth (tests/parity_util.py).  The tests marked ``gpu`` need an
H100; the reference self-checks and the coverage table run on the CPU.
"""
import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_fft_core_paths import _act, _at_offset, _par, core_inputs, core_ref
from tests.test_gpu_ragged import _exact_workspace
from tests.test_gpu_widths import NANS, _poison

gpu = pytest.mark.gpu
ROWS_PER_CALL = 16


# ------------------------------------------------------------------------------------------ per-row fp64 reference
def fftconv_pow2(u, k, D):
    """O.fftconv_ref with the transform padded to a power of two: the same linear convolution, without the slow transform
    lengths 2 (L - s_b) of arbitrary row slices."""
    L = u.shape[-1]
    n = 1 << (2 * L - 1).bit_length()
    return torch.fft.irfft(torch.fft.rfft(u, n=n) * torch.fft.rfft(k, n=n), n=n)[..., :L] + u * D.unsqueeze(-1)


def rows_core_ref(x, ib, sw, sb, k, fb, dy, starts, dtype=torch.float64, W=None, conv=fftconv_pow2):
    """core_ref on each row's slice [s_b, L), s_b clamped to [0, L] (a row with s_b >= L contributes nothing).

    x is p (B, 3D, L), or u (B, L, D) when W is given.  Returns y, c, dx (dp or du) and ds per row, zero at the pads;
    dk (D, L) as the sum of the rows' dk, each zero-padded to L; dib, dsw, dsb, dfb (and dW) summed over the rows."""
    B = x.shape[0]
    L = x.shape[1] if W is not None else x.shape[2]
    D = k.shape[0]
    z = lambda *s: torch.zeros(*s, dtype=dtype)
    out = dict(y=z(B, D, L), c=z(B, D, L), dx=z(*x.shape), ds=z(B, 3 * D, L), dk=z(D, L), dib=z(3 * D), dsw=z(3 * D, 3),
               dsb=z(3 * D), dfb=z(D))
    if W is not None:
        out["dW"] = z(*W.shape)
    for b, s in enumerate(starts):
        s = min(max(int(s), 0), L)
        if s >= L:
            continue
        n = L - s
        xs = x[b:b + 1, s:] if W is not None else x[b:b + 1, :, s:]
        r = core_ref(xs, ib, sw, sb, k[:, :n], fb, dy[b:b + 1, :, s:], dtype=dtype, W=W, conv=conv)
        for name in ("y", "c", "ds"):
            out[name][b, :, s:] = r[name][0]
        if W is not None:
            out["dx"][b, s:] = r["dx"][0]
        else:
            out["dx"][b, :, s:] = r["dx"][0]
        out["dk"][:, :n] += r["dk"]
        for name in ("dib", "dsw", "dsb", "dfb") + (("dW",) if W is not None else ()):
            out[name] += r[name]
    return out


def rows_core_refs(*args, **kw):
    """(fp32 reference, fp64 truth) of rows_core_ref on the host."""
    return rows_core_ref(*args, dtype=torch.float32, **kw), rows_core_ref(*args, dtype=torch.float64, **kw)


def masked_core(p, ib, sw, sb, k, fb, dy, starts, bug=None):
    """The masked core on the whole padded batch in fp64 autograd, masked where the *_ROWS kernels mask: pad samples of
    the short filters' input read 0 (no in_proj bias), g, c and y_pre are 0 at t < s_b.  ``bug`` plants one error:
      "start-1" / "start+1": every row's start off by one;
      "bias": pad samples of a window read the in_proj bias instead of 0;
      "x0": the x0 window unmasked (pad samples of p reach x0 at s_b and s_b + 1);
      "dc leak": dy_pre at the pads reaches dc (the forward values are unchanged: x - x.detach() adds an exact 0).
    Returns y, c and the gradients of p, ib, sw, sb, k, fb (names of core_ref)."""
    leaves = [t.detach().double().clone().requires_grad_(True) for t in (p, ib, sw, sb, k, fb)]
    p_, ib_, sw_, sb_, k_, fb_ = leaves
    B, C3, L = p.shape
    D = C3 // 3
    s = torch.tensor([int(v) for v in starts]) + {"start-1": -1, "start+1": 1}.get(bug, 0)
    keep = (torch.arange(L)[None, :] >= s[:, None])[:, None, :]
    P = p_ + ib_[None, :, None]
    Pin = torch.where(keep, P, ib_[None, :, None].expand_as(P) if bug == "bias" else torch.zeros_like(P))
    uc = O.short_filter(Pin, sw_.reshape(C3, 1, 3), sb_, L)
    x0, x1, v = uc.split(D, dim=1)
    if bug == "x0":
        x0 = O.short_filter(P, sw_.reshape(C3, 1, 3), sb_, L)[:, :D]
    g = torch.where(keep, v * x1, 0.0)
    c_raw = O.fftconv_ref(g, k_, fb_)
    c = torch.where(keep, c_raw, 0.0)
    y = torch.where(keep, c * x0, 0.0)
    if bug == "dc leak":
        y = y + (c_raw - c_raw.detach()) * x0.detach() * ~keep
    y.backward(dy.double())
    return dict(y=y.detach(), c=c.detach(), dx=p_.grad, dib=ib_.grad, dsw=sw_.grad, dsb=sb_.grad, dk=k_.grad,
                dfb=fb_.grad)


# ------------------------------------------------------------------------------------------ pads and row starts
def pad_mask(starts, L):
    """(B, 1, L) bool: True at the pads t < s_b."""
    return (torch.arange(L)[None, :] < torch.tensor([int(s) for s in starts])[:, None])[:, None, :]


def fill_pads(x, starts, fill, g):
    """x (B, C, L) with its pads replaced: "zero", an int seed (values of magnitude 3 to 10, random signs), one of the NaN
    encodings of tests/test_gpu_widths.NANS, or "inf" (random signs)."""
    pad = pad_mask(starts, x.shape[-1]).expand_as(x)
    if fill == "zero":
        v = torch.zeros_like(x)
    elif isinstance(fill, int):
        gs = torch.Generator().manual_seed(fill)
        v = (3 + 7 * torch.rand(x.shape, generator=gs)) * torch.randn(x.shape, generator=gs).sign()
    else:
        v = _poison(x, fill, g)
    return torch.where(pad, v, x)


def rows_inputs(B, D, L, starts, seed, fill=None, with_u=False):
    """core_inputs with the pads of p and dy_pre filled (large random values by default); u (with_u) is 0 at the pads."""
    t = core_inputs(B, D, L, seed, with_u=with_u)
    g = torch.Generator().manual_seed(seed + 1)
    fill = seed + 2 if fill is None else fill
    t["p"] = fill_pads(t["p"], starts, fill, g)
    t["dy"] = fill_pads(t["dy"], starts, fill, g)
    if with_u:
        t["u"] = torch.where(pad_mask(starts, L).transpose(1, 2), 0.0, t["u"])
    return t


def masked_geometry(L):
    """Where the masked passes cut a row of L samples.  Mirrors log_m_for and pick_log_m2 (csrc/api.cu) and ColGeo
    (csrc/fft_passes.cuh): M = 2^logM >= max(L, 1024) complex points with M2 = 1024 per column-FFT row, so row m1 holds
    the samples [2048 m1, 2048 m1 + 2048); a pass-1 / pass-3 CTA takes C columns of every row (C = 1024 for LOGM1 <= 3,
    512 for LOGM1 = 4, 256 / R2 with R2 = 2^(LOGM1 - 5) for the thread-group sizes, TWO); the staged epilogue of pass 3
    batches SB * R2 rows (SB = 8 forward, 4 backward); short_conv_bwd takes 8192 samples per CTA."""
    logm1 = max(10, (L - 1).bit_length()) - 10
    two = logm1 >= 5
    r2 = 1 << (logm1 - 5) if two else 1
    C = 256 // r2 if two else (1024 if logm1 <= 3 else 512)
    tiles = [t for m1 in range(-(-L // 2048)) for t in range(2048 * m1, 2048 * m1 + 2048, 2 * C) if 0 < t < L]
    b = dict(tile=tiles, row=list(range(2048, L, 2048)), span=list(range(8192, L, 8192)),
             batch_fwd=[t for t in [2048 * 8 * r2] if two and t < L], batch_bwd=[t for t in [2048 * 4 * r2] if two and t < L])
    return dict(logm1=logm1, two=two, r2=r2, C=C, boundaries=b)


def row_starts(L):
    """{0, 1, 2, 3, L-3, L-2, L-1} and boundary + {-2..2} for the first, a middle and the last tile boundary, the first
    and last column-FFT row boundary, the first staged-batch boundary of each epilogue, and the first, a middle and the
    last short_conv_bwd span, all kept to [0, L).  Past L = 2^17 the host reference of the long rows dominates the run
    time: there the first tile boundary stands for the boundaries near t = 0 (start 3, the first row and span edges and
    the middle ones are left out)."""
    b = masked_geometry(L)["boundaries"]
    long = L > 1 << 17
    picks = []
    for name, which in (("tile", (0, -1) if long else (0, None, -1)), ("row", (-1,) if long else (0, -1)),
                        ("batch_fwd", (0,)), ("batch_bwd", (0,)), ("span", (-1,) if long else (0, None, -1))):
        for i in which:
            if b[name]:
                picks.append(b[name][len(b[name]) // 2 if i is None else i])
    s = {0, 1, 2, L - 3, L - 2, L - 1} | ({3} if not long else set()) | {t + d for t in picks for d in range(-2, 3)}
    return sorted(v for v in s if 0 <= v < L)


def chunks(starts, n=ROWS_PER_CALL):
    return [starts[i:i + n] for i in range(0, len(starts), n)]


# one L with L % 4 == 0 and one odd L per transform template, and the tiny lengths of the 3-tap window
SWEEP_L = [1, 2, 3, 1000, 1023, 1536, 2047, 4096, 3001, 8192, 6145, 12288, 16383, 32768, 20001, 65532, 40001, 131072,
           100001, 262144, 160001, 524284, 300001, 1048576, 524289]


def decisions(L):
    """Cells of the coverage table a core_forward + core_backward call at L with row_start reaches."""
    g = masked_geometry(L)
    kind = "L%4==0" if L % 4 == 0 else ("odd" if L % 2 else "L%4==2")
    out = {("fwd", g["logm1"], kind), ("bwd", g["logm1"], kind), ("short_conv_bwd", "vec" if L % 2 == 0 else "scalar")}
    starts = set(row_starts(L))
    if g["two"] and kind == "L%4==0":          # cp.async staging: starts on the staged-batch edges and the tile halo
        b = g["boundaries"]
        if b["batch_fwd"][0] in starts and b["batch_bwd"][0] in starts:
            out.add(("staged batch", g["logm1"]))
        if all(b["tile"][0] + d in starts for d in (-2, -1, 0, 1, 2)):
            out.add(("tile halo", g["logm1"]))
    return out


# ------------------------------------------------------------------------------------------ CPU self-checks
def test_coverage_table():
    """The sweep reaches every LOGM1 in both masked directions with L % 4 == 0 (staged) and odd L (vec = 0), both
    short_conv_bwd variants, and on the TWO sizes starts on the staged-batch edges and on a tile edge's halo."""
    hit = set()
    for L in SWEEP_L:
        hit |= decisions(L)
        assert 0 < len(row_starts(L)) and all(0 <= s < L for s in row_starts(L))
    want = {(d, m, kind) for d in ("fwd", "bwd") for m in range(11) for kind in ("L%4==0", "odd")}
    want |= {("short_conv_bwd", "vec"), ("short_conv_bwd", "scalar")}
    want |= {(cell, m) for cell in ("staged batch", "tile halo") for m in range(5, 11)}
    assert not want - hit, f"table cells not hit: {sorted(want - hit, key=str)}"
    for L in (1, 2, 3):
        assert row_starts(L) == list(range(L))
    # the geometry: tile widths of ColGeo, and the first tile edge of a TWO size inside the first column row
    assert [masked_geometry(1 << (m + 10))["C"] for m in range(11)] == [1024] * 4 + [512, 256, 128, 64, 32, 16, 8]
    assert masked_geometry(1 << 20)["boundaries"]["tile"][:2] == [16, 32]


@pytest.mark.parametrize("L", [37, 130])
def test_rows_ref_all_starts_zero_is_core_ref(L):
    B, D = 3, 2
    t = core_inputs(B, D, L, seed=L)
    args = [t[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")]
    r = rows_core_ref(*args, [0] * B)
    f = core_ref(*args)
    for name in ("y", "c", "dx", "ds", "dk", "dib", "dsw", "dsb", "dfb"):
        torch.testing.assert_close(r[name], f[name], rtol=1e-12, atol=1e-12, msg=name)


@pytest.mark.parametrize("L", [9, 40, 333])
def test_rows_ref_direct_convolution_and_whole_batch_masking(L):
    """The per-row reference with its power-of-two FFT replaced by the O(L^2) time-domain sum or by O.fftconv_ref, and
    the masked core run on the whole padded batch (masked_core, masked where the kernels mask): the same outputs and
    gradients."""
    starts = [0, 1, 2, L // 2, L - 2, L - 1]
    t = rows_inputs(len(starts), 3, L, starts, seed=L, with_u=True)
    args = [t[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")]
    r = rows_core_ref(*args, starts)
    d = rows_core_ref(*args, starts, conv=O.fftconv_direct)
    f = rows_core_ref(*args, starts, conv=O.fftconv_ref)
    m = masked_core(*args, starts)
    for name in ("y", "c", "dx", "ds", "dk", "dib", "dsw", "dsb", "dfb"):
        torch.testing.assert_close(d[name], r[name], rtol=1e-10, atol=1e-10, msg=name)
        torch.testing.assert_close(f[name], r[name], rtol=1e-10, atol=1e-10, msg=f"fftconv_ref {name}")
        if name != "ds":
            torch.testing.assert_close(torch.where(pad_mask(starts, L), 0.0, m[name]) if name == "dx" else m[name],
                                       r[name], rtol=1e-10, atol=1e-10, msg=f"whole batch {name}")
    ru = rows_core_ref(t["u"], *args[1:], starts, W=t["W"])
    du = rows_core_ref(t["u"], *args[1:], starts, W=t["W"], conv=O.fftconv_direct)
    for name in ("y", "dx", "dW", "dib", "dk"):
        torch.testing.assert_close(du[name], ru[name], rtol=1e-10, atol=1e-10, msg=f"u {name}")


PLANTED = ["start-1", "start+1", "bias", "x0", "dc leak"]


@pytest.mark.parametrize("bug", PLANTED)
def test_parity_bar_rejects_planted_masking_bugs(bug):
    """Each planted masking bug is rejected by the bar against the correct fp32 / fp64 pair that the unplanted masked
    core passes.  A dc leak at the pads is exact arithmetic's no-op (g is 0 there, so neither dk, dfb nor dg at a real
    position pairs a pad dc with a non-zero operand): it shows once a pad of dy_pre is not finite, as the pad-contents
    test on the device feeds it."""
    L, D = 300, 3
    starts = [0, 1, 2, 3, 100, 255, 297, 299]
    t = rows_inputs(len(starts), D, L, starts, seed=5)
    if bug == "dc leak":
        t["dy"] = fill_pads(t["dy"], starts, "inf", torch.Generator().manual_seed(0))
    args = [t[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")]
    r32, r64 = rows_core_refs(*args, starts)
    pad = pad_mask(starts, L)
    n0 = len(PU._records)

    def bar(o):
        _act(o["y"], r32["y"], r64["y"], "y")
        _act(torch.where(pad, 0.0, o["dx"]), r32["dx"], r64["dx"], "dp")
        for name in ("dk", "dib", "dsw", "dsb", "dfb"):
            _par(o[name], r32[name], r64[name], name)

    try:
        bar(masked_core(*args, starts))
        with pytest.raises(AssertionError):
            bar(masked_core(*args, starts, bug=bug))
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


def _rows_run(H, t, starts, dev, p_off=0, kspec_off=False):
    """core_forward(save_c) with row_start, then core_backward twice on it: with dp (short_conv_bwd_rows_kernel) and with
    return_ds (rows_in_bias_grad).  p, dy_pre and c at p_off bytes past an aligned allocation; kspec one complex element
    off with kspec_off.  Returns every output on the host."""
    ib, sw, sb, k, fb = (t[n].to(dev) for n in ("ib", "sw", "sb", "k", "fb"))
    p, dy = t["p"].to(dev), t["dy"].to(dev)
    if p_off:
        p, dy = _at_offset(p, p_off), _at_offset(dy, p_off)
    rs = torch.tensor([int(s) for s in starts], dtype=torch.int32, device=dev)
    kspec = H.ops.filter_spectrum(k)
    if kspec_off:
        kspec = _at_offset(kspec, 8)
    o = {}
    o["y"], c, gs = H.ops.core_forward(p, ib, sw, sb, kspec, fb, True, rs)
    o["c"] = c
    if p_off:
        c = _at_offset(c, p_off)
    o["dp"], o["dk"], o["dsw"], o["dsb"], o["dfb"], o["dib"] = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs,
                                                                                   row_start=rs)
    o["ds"], o["dk_ds"], _, _, _, o["dib_ds"] = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs, return_ds=True,
                                                                    row_start=rs)
    torch.cuda.synchronize()
    return {n: v.cpu() for n, v in o.items()}


def _zero_at_pads(o, starts, tag, names=("y", "c", "dp", "ds")):
    L = o["y"].shape[-1]
    for n in names:
        pad = pad_mask(starts, L).expand_as(o[n])
        assert bool((o[n][pad] == 0).all()), f"{tag}: {n} is not exactly 0 at the pads"


def _check_rows(o, r32, r64, starts, tag):
    _act(o["y"], r32["y"], r64["y"], f"{tag} y_pre")
    _act(o["c"], r32["c"], r64["c"], f"{tag} c")
    _act(o["dp"], r32["dx"], r64["dx"], f"{tag} dp")
    _act(o["ds"], r32["ds"], r64["ds"], f"{tag} ds")
    for n in ("dk", "dsw", "dsb", "dfb", "dib"):
        _par(o[n], r32[n], r64[n], f"{tag} grad {n}")
    _par(o["dk_ds"], r32["dk"], r64["dk"], f"{tag} grad dk (return_ds)")
    _par(o["dib_ds"], r32["dib"], r64["dib"], f"{tag} grad dib (rows_in_bias_grad)")
    _zero_at_pads(o, starts, tag)


def _run_and_check(H, dev, D, L, starts, seed, tag, **kw):
    t = rows_inputs(len(starts), D, L, starts, seed)
    r32, r64 = rows_core_refs(*(t[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")), starts)
    o = _rows_run(H, t, starts, dev, **kw)
    _check_rows(o, r32, r64, starts, tag)
    return o


def _some_starts(L):
    """A dozen of row_starts(L) for the path tests: the edges and the first boundaries of each kind."""
    s = row_starts(L)
    return sorted(set(s[:6] + s[-3:] + s[len(s) // 2 - 1:len(s) // 2 + 2]))


# ------------------------------------------------------------------------------------------ 1. transform size sweep
@gpu
@pytest.mark.parametrize("L", SWEEP_L)
def test_rows_core_sweep(L):
    """Every masked mode at every LOGM1, row starts on every boundary kind of row_starts(L), D = 3, pads of p and dy_pre
    holding values of magnitude 3 to 10."""
    H = _H()
    dev = _dev()
    for i, starts in enumerate(chunks(row_starts(L))):
        _run_and_check(H, dev, 3, L, starts, seed=31 * L + i, tag=f"rows L={L} call {i}")


# ------------------------------------------------------------------------------------------ 2. fused route
@gpu
@pytest.mark.parametrize("L", [1000, 8188, 32764, 262140])          # LOGM1 = 0, 3, 5, 8
def test_rows_fused_route(L):
    """HyenaInCoreFn with row_start: u zero at the pads (its contract), dy_pre random there.  du at the real positions,
    dW and every other gradient against the per-row truth."""
    H = _H()
    dev = _dev()
    D = 3
    starts = _some_starts(L)
    t = rows_inputs(len(starts), D, L, starts, seed=37 * L, with_u=True)
    r32, r64 = rows_core_refs(t["u"], *(t[n] for n in ("ib", "sw", "sb", "k", "fb", "dy")), starts, W=t["W"])
    u, W, ib, sw, sb, k, fb = (t[n].to(dev).requires_grad_(True) for n in ("u", "W", "ib", "sw", "sb", "k", "fb"))
    rs = torch.tensor(starts, dtype=torch.int32, device=dev)
    y = H.ops.HyenaInCoreFn.apply(u, W, ib, sw.reshape(3 * D, 1, 3), sb, k, fb, None, rs)
    y.backward(t["dy"].to(dev))
    tag = f"rows fused L={L}"
    _act(y, r32["y"], r64["y"], f"{tag} y_pre")
    _zero_at_pads({"y": y.detach().cpu()}, starts, tag, ("y",))
    du = torch.where(pad_mask(starts, L).transpose(1, 2), 0.0, u.grad.cpu())
    _act(du, r32["dx"], r64["dx"], f"{tag} du")
    for n, got in dict(dW=W.grad, dib=ib.grad, dsw=sw.grad, dsb=sb.grad, dk=k.grad, dfb=fb.grad).items():
        _par(got, r32[n], r64[n], f"{tag} grad {n}")


# ------------------------------------------------------------------------------------------ 3. paths
# the left-padded prefills of tests/test_gpu_ragged.py at these lengths (rows of P, 517, 2, 1 and P, 3, P - 1, 40001)
REGISTER_STARTS = {1024: [0, 507, 1022, 1023], 65536: [0, 65533, 1, 25535]}


@gpu
@pytest.mark.parametrize("L", [1024, 30000, 65536, 120000, 400000])  # LOGM1 = 0, 5, 6, 7, 9, L % 4 == 0
def test_rows_register_path(L):
    """p, dy_pre and c 8 bytes off (vec = 1, no cp.async staging): the register path at sizes where staging would run."""
    starts = REGISTER_STARTS.get(L) or _some_starts(L)
    _run_and_check(_H(), _dev(), 3, L, starts, seed=41 * L, tag=f"rows register L={L}", p_off=8)


@gpu
@pytest.mark.parametrize("off", [4, 8])
def test_rows_operand_addresses(off):
    """p, dy_pre and c 4 bytes off (vec = 0) and 8 bytes off (vec, no staging) at a TWO size."""
    L = 40000
    _run_and_check(_H(), _dev(), 3, L, _some_starts(L), seed=43 + off, tag=f"rows p{off} L={L}", p_off=off)


@gpu
@pytest.mark.parametrize("kspec_off", [False, True])
def test_rows_batch_one(kspec_off):
    """B = 1 with the g spectrum saved: the staged ROW_CONV_BWD1, or with kspec one complex element off the unstaged one."""
    H = _H()
    dev = _dev()
    L = 40000
    for s in (0, 1, 2047, 2050, 16385, L - 1):
        _run_and_check(H, dev, 3, L, [s], seed=47 + s, tag=f"rows B=1 start {s} kspec8={kspec_off}", kspec_off=kspec_off)


@gpu
@pytest.mark.parametrize("L", [1000, 8188, 32764, 262140, 1048576])  # LOGM1 = 0, 3, 5, 8, 10
def test_rows_spectrum_recompute(monkeypatch, L):
    """HYENA_B200_SAVE_SPECTRUM=0: no saved g spectrum, so each backward recomputes g with COL_GATE_ROWS."""
    monkeypatch.setenv("HYENA_B200_SAVE_SPECTRUM", "0")
    H = _H()
    starts = _some_starts(L)
    if L == 1 << 20:
        starts = starts[:4] + starts[-4:]
    H._lib.profile_begin()
    _run_and_check(H, _dev(), 3, L, starts, seed=53 * L, tag=f"rows recompute L={L}")
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 3, prof          # the forward and the recomputation in each backward


@gpu
@pytest.mark.parametrize("L", [4096, 40000])
def test_rows_channel_groups(monkeypatch, L):
    """The workspace cut to 3 channels per launch (D = 7: 3 + 3 + 1, c0 > 0, a ragged last group), B = 5: every output
    against the per-row truth, the per-row outputs bit for bit those of the one-group run."""
    H = _H()
    dev = _dev()
    starts = [0, 1, 2047, 2050, L - 1]
    base = _run_and_check(H, dev, 7, L, starts, seed=59 * L, tag=f"rows groups L={L} one group")
    monkeypatch.setattr(H.ops, "workspace", _exact_workspace(H, 3))
    H._lib.profile_begin()
    got = _run_and_check(H, dev, 7, L, starts, seed=59 * L, tag=f"rows groups L={L} G=3")
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 3 and prof["col_fwd<dc>"][1] == 6, prof
    for n in ("y", "c", "dp", "ds", "dk"):
        assert torch.equal(got[n], base[n]), f"rows groups L={L}: {n} differs from the one-group run"


# ------------------------------------------------------------------------------------------ 4. pad contents
# sums reduced by atomicAdd across CTAs (pass 3 and short_conv_bwd; dib_ds follows from dsb): their summation order
# varies from run to run, so two runs may differ in the last bits, and two that agree once prove nothing
ATOMIC = ("dsw", "dsb", "dfb", "dib", "dib_ds")


@gpu
@pytest.mark.parametrize("L", [4097, 40000])
def test_rows_pad_contents(L):
    """The pads of p and dy_pre filled with zeros, two random seeds, the three NaN encodings and +-inf: y_pre, c, dp, ds
    and dk (no atomics) bit for bit the same, the atomic sums against the per-row fp64 truth for every fill, everything
    finite.  Every mask is a select, so a NaN pad never reaches an output."""
    H = _H()
    dev = _dev()
    D = 3
    starts = [0, 1, 2, 3, 2046, 2047, 2049, L // 2, L - 2, L - 1]
    t0 = rows_inputs(len(starts), D, L, starts, seed=67, fill="zero")
    r32, r64 = rows_core_refs(*(t0[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")), starts)
    zero = _rows_run(H, t0, starts, dev)
    _check_rows(zero, r32, r64, starts, f"rows pads zero L={L}")
    truth = {n: (r32[n], r64[n]) for n in ("dsw", "dsb", "dfb", "dib")}
    truth["dib_ds"] = truth["dib"]

    def run(fill):
        g = torch.Generator().manual_seed(71)
        t = dict(t0, p=fill_pads(t0["p"], starts, fill, g), dy=fill_pads(t0["dy"], starts, fill, g))
        return _rows_run(H, t, starts, dev)

    for fill in (1, 2, *NANS, "inf"):
        o = run(fill)
        tag = f"rows pads {fill} L={L}"
        for n, v in o.items():
            assert bool(torch.isfinite(v).all()), f"{tag}: non-finite {n}"
        for n in ("y", "c", "dp", "ds", "dk", "dk_ds"):
            assert torch.equal(o[n], zero[n]), f"{tag}: {n} differs from the run with zero pads"
        for n in ATOMIC:
            _par(o[n], *truth[n], f"{tag} grad {n}")


# ------------------------------------------------------------------------------------------ 5. out-of-range starts
@gpu
@pytest.mark.parametrize("L", [1000, 40000])
def test_rows_out_of_range_starts(L):
    """Starts -3, L and L + 5 among ordinary rows: a start <= 0 masks nothing (the plain core_fwd / core_bwd bits on its
    row), a start >= L masks the whole row (exact zeros), and the parameter gradients are the per-row truth without the
    fully masked rows."""
    H = _H()
    dev = _dev()
    D = 3
    starts = [-3, 0, L, 1, L + 5, L // 2]
    t = rows_inputs(len(starts), D, L, starts, seed=73)
    for b, s in enumerate(starts):              # a fully masked row holds large values everywhere
        if s >= L:
            t["p"][b] = fill_pads(t["p"][b:b + 1], [L], 7, None)[0]
            t["dy"][b] = fill_pads(t["dy"][b:b + 1], [L], 8, None)[0]
    r32, r64 = rows_core_refs(*(t[n] for n in ("p", "ib", "sw", "sb", "k", "fb", "dy")), starts)
    o = _rows_run(H, t, starts, dev)
    _check_rows(o, r32, r64, starts, f"rows out of range L={L}")
    ib, sw, sb, k, fb, p, dy = (t[n].to(dev) for n in ("ib", "sw", "sb", "k", "fb", "p", "dy"))
    kspec = H.ops.filter_spectrum(k)
    y, c, gs = H.ops.core_forward(p, ib, sw, sb, kspec, fb, True)
    dp = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs)[0]
    ds = H.ops.core_backward(dy, p, ib, sw, sb, kspec, fb, c, gs, return_ds=True)[0]
    plain = dict(y=y.cpu(), c=c.cpu(), dp=dp.cpu(), ds=ds.cpu())
    for b, s in enumerate(starts):
        for n in ("y", "c", "dp", "ds"):
            if s <= 0:
                assert torch.equal(o[n][b], plain[n][b]), f"L={L} start {s}: {n} differs from the plain core"
            elif s >= L:
                assert not o[n][b].any(), f"L={L} start {s}: {n} is not 0 on a fully masked row"
