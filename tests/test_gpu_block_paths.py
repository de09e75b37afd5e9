"""The residual-add + LayerNorm kernels' dispatch paths and the pre-norm Block / Backbone against fp64.

The host code of the block glue (csrc/k_layernorm.cu) picks a kernel per direction from the width and the alignment of
every operand, and a grid from the row count.  Each test below drives one family of those decisions on purpose and
compares every output with an fp64 truth through tests/parity_util.check:

| decision                                | selected by                                  | test                                   |
|-----------------------------------------|----------------------------------------------|----------------------------------------|
| fwd add_ln_fwd_kernel<NV>, NV 1 2 4 8   | D bucket (<= 128 NV); full and partial last  | test_sweep[w*]: D = 4 124 128 132 252  |
|                                         | float4 row per lane                          | 256 260 508 512 516 1020 1024          |
| bwd add_ln_bwd_kernel<NV>; > 48 KB smem | the same; opt-in for D > 768                 | the same widths                        |
| generic fwd / bwd by width              | D % 4 != 0 or D > 1024                       | test_sweep[w*]: D = 1 2 3 50 98 1028   |
|                                         |                                              | 2048 6144 6148 8192 (> 6144: the old   |
|                                         |                                              | generic bwd's smem limit)              |
| generic by alignment, per direction     | each operand's address                       | test_sweep[align*]: x, res, w, b off   |
|                                         |                                              | by 1 2 3 floats (fwd generic; bwd      |
|                                         |                                              | register unless w); test_raw_abi: dy,  |
|                                         |                                              | dres only (fwd register, bwd generic)  |
| grid capped, rows per warp > 1          | rows vs 64 * SMs (8 CTAs of 8 warps per SM)  | test_sweep[rows*]: 1 7 8 9, cap - 1,   |
|                                         |                                              | cap, cap + 1, 70000 on both paths;     |
|                                         |                                              | test_million_rows (2^20 at D = 256)    |
| optional operands                       | res / b / dres null                          | test_sweep (res None and present);     |
|                                         |                                              | test_raw_abi (b, dres null);           |
|                                         |                                              | test_block_bias_free_layernorm         |

Beyond the table: row statistics where LayerNorm kernels go wrong (constant rows, a 1e3 common offset, spread near
sqrt(eps); test_row_statistics), row isolation of NaN / inf (test_row_isolation), bitwise determinism of dx, dw, db at
70000 rows on every path (test_determinism), launch counts (test_launches) and whole-model training at sizes where every
warp handles many rows (test_backbone_training, test_block_bias_free_layernorm).

The fp32 twin (torch's F.layer_norm, or the oracle composition) is ``ref32`` and the fp64 truth ``ref64``, so any use of
the S8(c) hatch is book-kept.  The cap of the grid is read from the device; the coverage table counts it at 132 SMs
(H100 SXM).  The tests marked ``gpu`` need an H100; the self-checks of the truth, of the bar and of the table run on the
CPU.
"""
import math
from collections import namedtuple
from functools import partial

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_decode_paths import backbone_ref
from tests.test_gpu_widths import NANS, _act, _poison

gpu = pytest.mark.gpu

KWARPS = 8               # rows in flight per CTA (csrc/layernorm_args.h kWarps)
CTAS_PER_SM = 8          # ln_grid's cap (csrc/k_layernorm.cu)
SMS = 132                # H100 SXM: the SM count the coverage table assumes


# ------------------------------------------------------------------------------------------ the cases
Case = namedtuple("Case", "D rows res bias off")
REG_W = [4, 124, 128, 132, 252, 256, 260, 508, 512, 516, 1020, 1024]
GEN_W = [1, 2, 3, 50, 98, 1028, 2048, 6144, 6148, 8192]
ROWS = [1, 7, 8, 9, "cap-1", "cap", "cap+1", 70000]


def _sweep():
    out = {}
    for i, D in enumerate(REG_W + GEN_W):
        out[f"w{D}"] = Case(D, "cap+1" if D <= 2048 else 1000, i % 2 == 0, True, {})
    for D in (256, 50):
        for rows in ROWS:
            out[f"rows{rows}_D{D}"] = Case(D, rows, True, True, {})
    for name in ("x", "res", "w", "b"):
        for k in (1, 2, 3):
            out[f"align_{name}{k}"] = Case(256, "cap+1", True, True, {name: k})
    return out


SWEEP = _sweep()
# raw ABI: (D, rows, bias, dres, offsets): the backward alone on an unaligned dy / dres, and null b / dres
RAW = {"dy1": Case(256, "cap+1", True, True, {"dy": 1}), "dy3": Case(1024, "cap+1", True, True, {"dy": 3}),
       "dres2": Case(256, "cap+1", True, True, {"dres": 2}), "nulls_D260": Case(260, "cap+1", False, False, {}),
       "nulls_D98": Case(98, "cap+1", False, False, {})}
DETERMINISM = {"D256": (256, {}), "D1024": (1024, {}), "D50": (50, {}), "D2048": (2048, {}), "D6148": (6148, {}),
               "dy_unaligned": (256, {"dy": 1})}
DET_ROWS = 70000


def cap(sms):
    return CTAS_PER_SM * sms * KWARPS


def resolve(rows, sms):
    if isinstance(rows, int):
        return rows
    return cap(sms) + {"cap-1": -1, "cap": 0, "cap+1": 1}[rows]


def _grid(rows, sms):
    return min(max(-(-rows // KWARPS), 1), CTAS_PER_SM * sms)


def _nv(D):
    return 1 if D <= 128 else 2 if D <= 256 else 4 if D <= 512 else 8


def paths(D, off):
    """(forward path, backward path): NV of the register kernel or "generic" (launch_add_ln_fwd / _bwd)."""
    width_ok = D % 4 == 0 and D <= 1024
    fwd_ok = width_ok and not any(off.get(n, 0) % 4 for n in ("x", "res", "w", "b"))
    bwd_ok = width_ok and not any(off.get(n, 0) % 4 for n in ("dy", "dres", "w"))
    return (_nv(D) if fwd_ok else "generic"), (_nv(D) if bwd_ok else "generic")


def decisions(c, sms=SMS, raw=False):
    rows = resolve(c.rows, sms)
    fp, bp = paths(c.D, c.off)
    hit = {("fwd", fp), ("bwd", bp), ("res", c.res), ("b", c.bias), ("raw", raw)}
    if raw:
        hit.add(("dres", c.bias))               # RAW cases pass dres exactly when they pass b
    if bp != "generic":
        hit.add(("bwd smem opt-in", c.D > 768))
    if fp != "generic":
        hit.add(("bucket fill", fp, "full" if c.D == 128 * fp else "partial"))
    if c.D % 4:
        hit.add(("generic", "D % 4"))
    if c.D > 1024:
        hit.add(("generic", "D > 1024"))
    if c.D > 6144:
        hit.add(("generic", "D > 6144"))
    for n, k in c.off.items():
        hit.add(("offset", n, k))
    if (fp == "generic") != (bp == "generic"):
        hit.add(("mixed", "fwd generic" if fp == "generic" else "bwd generic"))
    g = _grid(rows, sms)
    hit |= {("rows", c.rows), ("grid capped", g == CTAS_PER_SM * sms)}
    if rows > g * KWARPS:
        hit |= {("rows per warp > 1", "register" if fp != "generic" else "generic")}
    return hit


def test_coverage_table():
    """Every cell of the module docstring's table is hit by the cases above."""
    hit = set()
    for c in SWEEP.values():
        hit |= decisions(c)
    for c in RAW.values():
        hit |= decisions(c, raw=True)
    want = {(d, nv) for d in ("fwd", "bwd") for nv in (1, 2, 4, 8, "generic")}
    want |= {("bwd smem opt-in", True), ("bwd smem opt-in", False)}
    want |= {("bucket fill", nv, f) for nv in (1, 2, 4, 8) for f in ("full", "partial")}
    want |= {("generic", why) for why in ("D % 4", "D > 1024", "D > 6144")}
    want |= {("offset", n, k) for n in ("x", "res", "w", "b") for k in (1, 2, 3)} | {("offset", "dy", 1),
                                                                                       ("offset", "dres", 2)}
    want |= {("mixed", "fwd generic"), ("mixed", "bwd generic")}
    want |= {("rows", r) for r in ROWS} | {("grid capped", True), ("grid capped", False)}
    want |= {("rows per warp > 1", "register"), ("rows per warp > 1", "generic")}
    want |= {("res", True), ("res", False), ("b", False), ("dres", False)}
    assert not want - hit, f"table cells not hit: {sorted(want - hit, key=str)}"
    # the bucket edges the table names: one past each edge holds a partial last float4 row
    assert {132, 260, 516} <= {c.D for c in SWEEP.values() if paths(c.D, c.off)[0] != "generic"}
    # cap - 1 and cap fill the grid with one row per warp; cap + 1 gives a warp a second row
    for rows, more in (("cap-1", False), ("cap", False), ("cap+1", True)):
        r = resolve(rows, SMS)
        assert (r > _grid(r, SMS) * KWARPS) == more


# ------------------------------------------------------------------------------------------ fp64 truth and the bar
def ln_formula(x, res, w, b, dy, dres, eps, bug=None, sms=SMS):
    """The fused op in closed form, in the dtype of its arguments: y, res_out, dx, dw, db (db None without b).  ``bug``
    applies one of BUGS (the bar's self-check)."""
    r = x + res if res is not None else x
    rows, D = r.shape
    mean = r.mean(-1, keepdim=True)
    var = ((r - mean) ** 2).sum(-1, keepdim=True) / (D - 1 if bug == BUGS[0] else D)
    if bug == BUGS[2]:
        r32 = r.float()
        var = ((r32 * r32).mean(-1, keepdim=True) - r32.mean(-1, keepdim=True) ** 2).to(r.dtype)
    rstd = 1 / (var.sqrt() + eps) if bug == BUGS[1] else (var + eps).rsqrt()
    xh = (r - mean) * rstd
    ww = w.clone()
    if bug == BUGS[6]:
        t = D - D % 4
        ww[t:] = w[t - 1:D - 1]
    y = xh * ww + (b if b is not None else 0)
    g = dy * ww
    m1 = g.mean(-1, keepdim=True)
    m2 = (g * xh).mean(-1, keepdim=True)
    dx = rstd * (g - m1 - (0 if bug == BUGS[5] else xh * m2))
    if dres is not None and bug != BUGS[4]:
        dx = dx + dres
    keep = slice(0, rows)
    if bug == BUGS[3]:
        keep = slice(0, (-(-rows // cap(sms)) - 1) * cap(sms))
    dw = (dy * xh)[keep].sum(0)
    db = dy[keep].sum(0) if b is not None else None
    return y, (res if bug == BUGS[7] else r), dx, dw, db


def test_formula_matches_autograd():
    """ln_formula (no bug) is torch's own LayerNorm and its autograd in fp64, with and without res / b / dres."""
    g = torch.Generator().manual_seed(0)
    rows, D = 300, 98
    x, res, dy, dres = (torch.randn(rows, D, generator=g, dtype=torch.float64) for _ in range(4))
    w = 1 + 0.5 * torch.randn(D, generator=g, dtype=torch.float64)
    b = 0.5 * torch.randn(D, generator=g, dtype=torch.float64)
    for rr, bb, dd in ((res, b, dres), (None, None, None)):
        xx, ww = x.clone().requires_grad_(), w.clone().requires_grad_()
        bl = bb.clone().requires_grad_() if bb is not None else None
        r = xx + rr if rr is not None else xx
        y = F.layer_norm(r, (D,), ww, bl, 1e-5)
        torch.autograd.backward((y, r), (dy, dd if dd is not None else torch.zeros_like(dy)))
        fy, fr, fdx, fdw, fdb = ln_formula(x, rr, w, bb, dy, dd, 1e-5)
        for a, e in ((fy, y), (fr, r), (fdx, xx.grad), (fdw, ww.grad)) + (((fdb, bl.grad),) if bb is not None else ()):
            torch.testing.assert_close(a, e.detach(), rtol=1e-12, atol=1e-12)


def _stat_rows(rows, D, eps, kinds, g):
    """Rows of the given kinds in turn: "unit" N(0, 1); "const" a constant (exact in fp32, so is the row's mean at a
    power-of-two D); "offset" 1e3 + N(0, 1) on a 1/8 grid (its sum is exact in fp32 up to D = 2048, so the two-pass mean
    is too); "tiny" sqrt(eps) * N(0, 1), a spread near the epsilon."""
    x = torch.randn(rows, D, generator=g)
    consts = torch.tensor([0.75, -3.5, 1e3, 0.0])
    for i, kind in enumerate(kinds):
        sel = slice(i, rows, len(kinds))
        n = x[sel].shape[0]
        if kind == "const":
            x[sel] = consts[torch.arange(n) % 4][:, None].expand(n, D)
        elif kind == "offset":
            x[sel] = 1e3 + torch.round(torch.randn(n, D, generator=g) * 8) / 8
        elif kind == "tiny":
            x[sel] = math.sqrt(eps) * torch.randn(n, D, generator=g)
    return x


BUGS = ["variance divided by D - 1", "eps outside the square root", "one-pass fp32 variance",
        "dw / db miss the rows of the last grid-stride pass", "dres not added to dx", "mean(g xhat) term dropped",
        "tail columns take the neighbouring column's w", "res_out returns res instead of x + res"]
BUG_OUT = dict(zip(BUGS, ["y", "y", "y", "dw", "dx", "dx", "y", "r"]))


@pytest.mark.parametrize("bug", BUGS)
def test_parity_bar_rejects_layernorm_bugs(bug):
    """Each bug, applied to the fp64 truth, is rejected by the bar that the unperturbed truth passes.  The rows mix the
    statistics of test_row_statistics; D = 98 has a D % 4 tail; 9001 rows on 132 SMs need a second grid-stride pass."""
    rows, D, eps = 9001, 98, 1e-5
    g = torch.Generator().manual_seed(BUGS.index(bug))
    x = _stat_rows(rows, D, eps, ["unit", "offset", "tiny", "const"], g).double()
    res = torch.randn(rows, D, generator=g, dtype=torch.float64) * 1e-3
    w = 1 + 0.5 * torch.randn(D, generator=g, dtype=torch.float64)
    b = 0.5 * torch.randn(D, generator=g, dtype=torch.float64)
    dy, dres = (torch.randn(rows, D, generator=g, dtype=torch.float64) for _ in range(2))
    names = ["y", "r", "dx", "dw", "db"]
    truth = dict(zip(names, ln_formula(x, res, w, b, dy, dres, eps)))
    wrong = dict(zip(names, ln_formula(x, res, w, b, dy, dres, eps, bug=bug)))
    out = BUG_OUT[bug]
    pg = out in ("dw", "db")
    n0 = len(PU._records)
    try:
        PU.check(truth[out].float(), truth[out].float(), "unperturbed", ref64=truth[out], param_grad=pg)
        with pytest.raises(AssertionError):
            PU.check(wrong[out], truth[out].float(), bug, ref64=truth[out], param_grad=pg)
    finally:
        del PU._records[n0:]            # self-checks of the bar, not parity records


def test_block_rejects_non_affine_layernorm():
    """The fused kernel reads the norm's weight (and bias): a LayerNorm without them is refused at construction."""
    import hyena_dna_b200 as H

    def mixer(d):
        return nn.Identity()

    with pytest.raises(H.HyenaB200Error):
        H.Block(16, mixer_cls=mixer, norm_cls=partial(nn.LayerNorm, elementwise_affine=False))
    H.Block(16, mixer_cls=mixer, norm_cls=partial(nn.LayerNorm, bias=False))      # no bias is fine


# ------------------------------------------------------------------------------------------ device helpers
def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _make(shape, off, name, g, scale=1.0, shift=0.0):
    """A contiguous random tensor that starts ``off[name]`` floats into its allocation (16-byte aligned iff 0 mod 4)."""
    k = off.get(name, 0)
    buf = torch.randn(math.prod(shape) + k, generator=g, device="cuda") * scale + shift
    t = buf[k:].view(shape)
    assert (t.data_ptr() % 16 == 0) == (k % 4 == 0)
    return t


def _inputs(c, rows, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D, off = c.D, c.off
    x = _make((rows, D), off, "x", g)
    res = _make((rows, D), off, "res", g, 3.0) if c.res else None
    w = _make((D,), off, "w", g, 0.5, 1.0)
    b = _make((D,), off, "b", g, 0.5) if c.bias else None
    dy = _make((rows, D), off, "dy", g)
    dres = _make((rows, D), off, "dres", g)
    return x, res, w, b, dy, dres


def _twin(x, res, w, b, dy, dres, eps, dtype, lo, hi, leaves):
    """torch's LayerNorm + autograd in ``dtype`` on rows [lo, hi): y, res_out, dx; dw / db accumulate into ``leaves``."""
    xx = x[lo:hi].to(dtype, copy=True).requires_grad_(True)
    r = xx + res[lo:hi].to(dtype) if res is not None else xx
    y = F.layer_norm(r, (x.shape[1],), leaves[0], leaves[1], eps)
    torch.autograd.backward((y, r), (dy[lo:hi].to(dtype),
                                     dres[lo:hi].to(dtype) if dres is not None else torch.zeros_like(r)))
    return y.detach(), r.detach(), xx.grad


def _compare(ours, x, res, w, b, dy, dres, eps, what, chunk=None):
    """ours = (y, res_out, dx, dw, db) against the fp32 twin and the fp64 truth, by row chunks of ``chunk``."""
    rows = x.shape[0]
    chunk = chunk or rows
    lv = {dt: (w.detach().to(dt, copy=True).requires_grad_(True),
               b.detach().to(dt, copy=True).requires_grad_(True) if b is not None else None)
          for dt in (torch.float32, torch.float64)}
    for lo in range(0, rows, chunk):
        hi = min(lo + chunk, rows)
        tag = what if chunk >= rows else f"{what} rows [{lo}, {hi})"
        t32 = _twin(x, res, w, b, dy, dres, eps, torch.float32, lo, hi, lv[torch.float32])
        t64 = _twin(x, res, w, b, dy, dres, eps, torch.float64, lo, hi, lv[torch.float64])
        for i, name in enumerate(("y", "res_out", "dx")):
            PU.check(ours[i][lo:hi], t32[i], f"{tag} {name}", ref64=t64[i])
        del t32, t64
    PU.check(ours[3], lv[torch.float32][0].grad, f"{what} dw", ref64=lv[torch.float64][0].grad, param_grad=True)
    if b is not None:
        PU.check(ours[4], lv[torch.float32][1].grad, f"{what} db", ref64=lv[torch.float64][1].grad, param_grad=True)


def _run_ops(x, res, w, b, dy, dres, eps):
    """ops.add_layer_norm forward + backward on leaves that keep the operands' addresses."""
    H = _H()
    xl = x.detach().requires_grad_(True)
    rl = res.detach().requires_grad_(True) if res is not None else None
    wl = w.detach().requires_grad_(True)
    bl = b.detach().requires_grad_(True) if b is not None else None
    y, r = H.ops.add_layer_norm(xl, rl, wl, bl, eps)
    torch.autograd.backward((y, r), (dy, dres))
    if rl is not None:
        assert torch.equal(rl.grad.view(torch.int32), xl.grad.view(torch.int32))   # the residual's gradient is the input's
    return y.detach(), r.detach(), xl.grad, wl.grad, (bl.grad if bl is not None else None)


def _raw_fwd(x, res, w, b, eps):
    H = _H()
    rows, D = x.shape
    y, ro = torch.empty(rows, D, device=x.device), torch.empty(rows, D, device=x.device)
    mean, rstd = torch.empty(rows, device=x.device), torch.empty(rows, device=x.device)
    p = H.ops._ptr
    H._lib.check(H._lib.lib().hyena_b200_add_layernorm_fwd(p(x), p(res), p(w), p(b), float(eps), p(ro), p(y), p(mean),
                                                           p(rstd), rows, D, H.ops._stream()))
    return y, ro, mean, rstd


def _raw_bwd(dy, dres, r, w, mean, rstd, with_db):
    H = _H()
    rows, D = r.shape
    need = int(H._lib.lib().hyena_b200_add_layernorm_scratch_bytes(rows, D))
    sc = torch.empty(need, dtype=torch.uint8, device=r.device)
    dx = torch.empty(rows, D, device=r.device)
    dw = torch.empty(D, device=r.device)
    db = torch.empty(D, device=r.device) if with_db else None
    p = H.ops._ptr
    H._lib.check(H._lib.lib().hyena_b200_add_layernorm_bwd(p(dy), p(dres), p(r), p(w), p(mean), p(rstd), p(dx), p(dw),
                                                           p(db), rows, D, p(sc), need, H.ops._stream()))
    return dx, dw, db


# ------------------------------------------------------------------------------------------ 1. the fp64 sweep
@gpu
@pytest.mark.parametrize("name", list(SWEEP))
def test_sweep(name):
    """ops.add_layer_norm forward + backward: y, res_out, dx (= the residual's gradient), dw, db against fp64."""
    _dev()
    c = SWEEP[name]
    rows = resolve(c.rows, _sms())
    ins = _inputs(c, rows, seed=len(name) * 1000 + c.D)
    ours = _run_ops(*ins, 1e-5)
    _compare(ours, *ins, 1e-5, name)


@gpu
def test_million_rows():
    """2^20 rows at D = 256, about 124 rows per warp on 132 SMs: the benchmark's B * L.  The truth is taken in row
    chunks, dw / db accumulated in fp64."""
    _dev()
    c = Case(256, 1 << 20, False, True, {})
    ins = _inputs(c, c.rows, seed=20)
    ours = _run_ops(*ins, 1e-5)
    assert torch.equal(ours[1], ins[0])                 # no residual: res_out is x
    _compare(ours, *ins, 1e-5, "2^20 rows", chunk=1 << 17)


@gpu
@pytest.mark.parametrize("name", list(RAW))
def test_raw_abi(name):
    """hyena_b200_add_layernorm_fwd / _bwd called directly: a backward whose only unaligned operand is dy or dres (its
    forward on the register path), and null b and dres."""
    _dev()
    c = RAW[name]
    rows = resolve(c.rows, _sms())
    x, res, w, b, dy, dres = _inputs(c, rows, seed=len(name))
    if not c.bias:
        dres = None
    y, ro, mean, rstd = _raw_fwd(x, res, w, b, 1e-5)
    dx, dw, db = _raw_bwd(dy, dres, ro, w, mean, rstd, c.bias)
    _compare((y, ro, dx, dw, db), x, res, w, b, dy, dres, 1e-5, f"raw {name}")


# ------------------------------------------------------------------------------------------ 2. row statistics
STATS = [(256, ["const", "offset", "tiny", "unit"]), (2048, ["const", "offset", "tiny", "unit"]),
         (260, ["tiny", "unit"]), (98, ["tiny", "unit"])]


@gpu
@pytest.mark.parametrize("eps", [1e-5, 1e-6, 1e-12])
@pytest.mark.parametrize("D,kinds", STATS, ids=[f"D{d}" for d, _ in STATS])
def test_row_statistics(D, kinds, eps):
    """Constant rows (variance 0), rows at a 1e3 common offset (a one-pass E[x^2] - E[x]^2 variance loses every digit)
    and rows whose spread is near sqrt(eps), on the register path (256, 260) and the generic one (2048, 98).  The inputs
    keep the row means exact in fp32 (see _stat_rows), so the fp32 reference is the fp64 truth rounded to fp32: torch's
    fp32 LayerNorm rounds the mean of the offset rows, which is not what is under test.  Each row kind is checked on its
    own, activations at their own scale (_act): dx of a row is rstd times unit-scale terms, up to 1e6 at eps = 1e-12."""
    dev = _dev()
    rows = cap(_sms()) + 1
    g = torch.Generator().manual_seed(D)
    x = _stat_rows(rows, D, eps, kinds, g).to(dev)
    w = (1 + 0.5 * torch.randn(D, generator=g)).to(dev)
    b = (0.5 * torch.randn(D, generator=g)).to(dev)
    dy, dres = (torch.randn(rows, D, generator=g).to(dev) for _ in range(2))
    ours = _run_ops(x, None, w, b, dy, dres, eps)
    truth = ln_formula(x.double(), None, w.double(), b.double(), dy.double(), dres.double(), eps)
    tag = f"stats D={D} eps={eps:g}"
    for i, kind in enumerate(kinds):
        for got, t, name in zip(ours[:3], truth[:3], ("y", "res_out", "dx")):
            _act(got[i::len(kinds)], t[i::len(kinds)].float(), t[i::len(kinds)], f"{tag} {kind} rows {name}")
    for got, t, name in zip(ours[3:], truth[3:], ("dw", "db")):
        PU.check(got, t.float(), f"{tag} {name}", ref64=t, param_grad=True)
    if "const" in kinds:
        assert torch.equal(ours[0][0::4], b.expand(ours[0][0::4].shape)), "constant rows: y is not exactly b"


# ------------------------------------------------------------------------------------------ 3. row isolation
KINDS = [*NANS, "inf"]


@gpu
@pytest.mark.parametrize("D", [256, 50])
def test_row_isolation(D):
    """One row of x, then of dy, all NaN (three encodings) or all +-inf: every other row's y, res_out and dx are the
    bits of a clean run, and the poisoned row's are non-finite (dw / db sum over rows and are left out)."""
    dev = _dev()
    rows, bad = cap(_sms()) + 1000, 4321
    c = Case(D, rows, True, True, {})
    x, res, w, b, dy, dres = _inputs(c, rows, seed=D)
    clean = _run_ops(x, res, w, b, dy, dres, 1e-5)
    keep = torch.ones(rows, dtype=torch.bool, device=dev)
    keep[bad] = False
    for kind in KINDS:
        for where in ("x", "dy"):
            g = torch.Generator(device=dev).manual_seed(7)
            x2, dy2 = x.clone(), dy.clone()
            t = x2 if where == "x" else dy2
            t[bad] = _poison(t[bad], kind, g)
            y, r, dx, _, _ = _run_ops(x2, res, w, b, dy2, dres, 1e-5)
            for got, want, name in ((y, clean[0], "y"), (r, clean[1], "res_out"), (dx, clean[2], "dx")):
                assert torch.equal(got[keep], want[keep]), f"D={D} {kind} in {where}: {name} of other rows changed"
            assert not bool(torch.isfinite(dx[bad]).any()), f"D={D} {kind} in {where}: finite dx in the poisoned row"
            if where == "x":
                assert not bool(torch.isfinite(y[bad]).any()), f"D={D} {kind}: finite y in the poisoned row"


# ------------------------------------------------------------------------------------------ 4. determinism, launches
@gpu
@pytest.mark.parametrize("name", list(DETERMINISM))
def test_determinism(name):
    """Two backward runs at 70000 rows (every warp handles several rows) give the same bits of dx, dw and db: register
    path (256, 1024), generic path by width (50, 2048, 6148) and by an unaligned dy."""
    dev = _dev()
    D, off = DETERMINISM[name]
    assert DET_ROWS > 2 * cap(_sms())
    g = torch.Generator(device=dev).manual_seed(D)
    r = torch.randn(DET_ROWS, D, generator=g, device=dev)
    dy = _make((DET_ROWS, D), off, "dy", g)
    w = 1 + 0.5 * torch.randn(D, generator=g, device=dev)
    var, mean = torch.var_mean(r, dim=1, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    a = _raw_bwd(dy, None, r, w, mean, rstd, True)
    bb = _raw_bwd(dy, None, r, w, mean, rstd, True)
    for u, v, what in zip(a, bb, ("dx", "dw", "db")):
        assert torch.equal(u, v), f"{name}: {what} differs between two runs"
    if D == 6148:        # past the 48 KB of shared memory the generic backward once asked for: also right
        truth = ln_formula(r[:2000].double(), None, w.double(), None, dy[:2000].double(), None, 1e-5)
        PU.check(a[0][:2000], truth[2].float(), f"determinism {name} dx", ref64=truth[2])


@gpu
@pytest.mark.parametrize("D", [256, 98])
def test_launches(D):
    """One launch forward, two backward (the kernel and the fixed-order reduction of its partials), on either path."""
    dev = _dev()
    H = _H()
    x = torch.randn(1000, D, device=dev, requires_grad=True)
    w = torch.randn(D, device=dev, requires_grad=True)
    b = torch.randn(D, device=dev, requires_grad=True)
    H._lib.profile_begin()
    y, r = H.ops.add_layer_norm(x, None, w, b, 1e-5)
    prof = H._lib.profile_end()
    assert set(prof) == {"add_layer_norm"} and prof["add_layer_norm"][1] == 1, prof
    H._lib.profile_begin()
    y.sum().backward()
    prof = H._lib.profile_end()
    assert set(prof) == {"add_layer_norm"} and prof["add_layer_norm"][1] == 2, prof


# ------------------------------------------------------------------------------------------ 5. Backbone / Block training
def _ln_randomize(m, g):
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.LayerNorm):
                mod.weight.copy_(1 + 0.3 * torch.randn(mod.weight.shape, generator=g))
                if mod.bias is not None:
                    mod.bias.copy_(0.3 * torch.randn(mod.bias.shape, generator=g))
            if isinstance(mod, _H().HyenaOperator):
                mod.in_proj.bias.copy_(0.02 * torch.randn(mod.in_proj.bias.shape, generator=g))


def _leaves(m, dev, dtype):
    names = {n for n, _ in m.named_parameters()}
    return {k: v.detach().to(dev, dtype, copy=True).requires_grad_(k in names) for k, v in m.state_dict().items()}


def _check_grads(m, ref, what):
    for n, p in m.named_parameters():
        assert p.grad is not None, f"{what}: no gradient for {n}"
        PU.check(p.grad, ref[32][n].grad, f"{what} grad {n}", ref64=ref[64][n].grad, param_grad=True)


BACKBONES = {"B2_L32768_D256_mlp": (2, 1 << 15, 256, 2, True), "B1_L20000_D98_mlp": (1, 20000, 98, 2, True),
             "B3_L4097_D516": (3, 4097, 516, 1, False)}


@gpu
@pytest.mark.parametrize("name", list(BACKBONES))
def test_backbone_training(name):
    """Backbone forward + backward against an fp64 composition of its own parameters (backbone_ref through the oracle
    operator): y, dx and every named parameter's gradient, norm1 / norm2 / ln_f weight and bias included.  Row counts
    past the grid cap, so the add + LayerNorm kernels run several rows per warp on each path.  Activations are held to
    the bar with the absolute term at their own scale (_act, as for the operator in tests/test_gpu_widths.py)."""
    H = _H()
    dev = _dev()
    B, L, D, n_layer, with_mlp = BACKBONES[name]
    g = torch.Generator().manual_seed(L + D)
    torch.manual_seed(L + D)
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh")) if with_mlp else None
    m = H.Backbone(D, n_layer, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    _ln_randomize(m, g)
    m = m.to(dev)
    x = torch.randn(B, L, D, generator=g)
    dy = torch.randn(B, L, D, generator=g)
    xg = x.to(dev).requires_grad_(True)
    y = m(xg)
    y.backward(dy.to(dev))
    ref, out = {}, {}
    for bits, dt in ((32, torch.float32), (64, torch.float64)):
        ref[bits] = _leaves(m, dev, dt)
        xx = x.to(dev, dt).requires_grad_(True)
        yy = backbone_ref(xx, ref[bits], n_layer, dt)
        yy.backward(dy.to(dev, dt))
        out[bits] = (yy.detach(), xx.grad)
        del yy, xx
    _act(y, out[32][0], out[64][0], f"backbone {name} y")
    _act(xg.grad, out[32][1], out[64][1], f"backbone {name} dx")
    _check_grads(m, ref, f"backbone {name}")


@gpu
def test_block_bias_free_layernorm():
    """A Block whose LayerNorm has no bias, with an incoming residual that requires grad: the hidden and residual
    outputs, dx, dres and every parameter gradient against an fp64 composition."""
    H = _H()
    dev = _dev()
    B, L, D = 2, 5000, 132
    g = torch.Generator().manual_seed(132)
    torch.manual_seed(132)
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    blk = H.Block(D, mixer_cls=mixer, norm_cls=partial(nn.LayerNorm, bias=False))
    assert blk.norm1.bias is None
    _ln_randomize(blk, g)
    blk = blk.to(dev)
    x, res, dy, dres = (torch.randn(B, L, D, generator=g) for _ in range(4))
    xg, rg = x.to(dev).requires_grad_(True), res.to(dev).requires_grad_(True)
    h, r = blk(xg, rg)
    torch.autograd.backward((h, r), (dy.to(dev), dres.to(dev)))
    ref, out = {}, {}
    for bits, dt in ((32, torch.float32), (64, torch.float64)):
        S = ref[bits] = _leaves(blk, dev, dt)
        xx, rr = x.to(dev, dt).requires_grad_(True), res.to(dev, dt).requires_grad_(True)
        rs = xx + rr
        hn = F.layer_norm(rs, (D,), S["norm1.weight"], None, 1e-5)
        P = O.canonical({k[len("mixer."):]: v for k, v in S.items() if k.startswith("mixer.")})
        hh = O.hyena_operator(hn, P)
        torch.autograd.backward((hh, rs), (dy.to(dev, dt), dres.to(dev, dt)))
        out[bits] = (hh.detach(), rs.detach(), xx.grad, rr.grad)
    for i, what in enumerate(("hidden", "residual", "dx", "dres")):
        got = (h, r, xg.grad, rg.grad)[i]
        _act(got, out[32][i], out[64][i], f"bias-free block {what}")
    _check_grads(blk, ref, "bias-free block")
