"""The windowed FFT core of the streaming forward against fp64: the *_WIN modes at every transform size.

``hyena_b200_core_fwd_windows`` runs COL_GATE_PACKED and INV_CONV_FWD_WIN (the order-2 core), and
``hyena_b200_fftconv_fwd_windows`` runs COL_PLAIN_WIN and INV_PLAIN_FWD_WIN (the plain convolution of every order >= 3
recurrence), once per set of window rows of one length L_b (DESIGN.md section 4.21).  Window row b reads a packed
tensor at seg_base[b] + t for t in [row_start[b], L_b) only and stores its outputs at t >= max(out_start[b],
row_start[b]) only: the positions before are its context, whose outputs another window stores.  The tests drive both
entry points directly (``windows_run``, which mirrors ops.core_forward_windows / fftconv_forward_windows but owns its
output buffer, pre-filled with SENTINEL, so every position no window owns can be checked), with hand-made seg_base /
row_start / out_start tables (the C ABI accepts any L <= 2^20, any start and any out_start).

Truth is per window: a window is a packed sequence of its positions [rs, L_b) whose outputs are kept from max(os, rs),
so ``window_ref`` runs the fp64 core (tests/test_gpu_fft_core_paths.core_ref, k cut to L_b - rs) or the plain
convolution with its D skip term (tests/test_gpu_rows_core_paths.fftconv_pow2) on that slice alone, with its fp32 twin,
and scatters only the stored range.  Every layout keeps the stored ranges of its windows disjoint, and every table keeps
seg_base + t inside the buffer for t >= row_start.

| decision                                                      | selected by                    | test                              |
|---------------------------------------------------------------|--------------------------------|-----------------------------------|
| INV_CONV_FWD_WIN and COL_GATE_PACKED (through core_fwd_windows) | L_b, LOGM1 = 0..10           | test_window_sweep[core-*], test_window_abi_lengths[core-*] |
| COL_PLAIN_WIN and INV_PLAIN_FWD_WIN, LOGM1 = 0..10            | L_b                            | test_window_sweep[plain-*], test_window_abi_lengths[plain-*] |
| odd L, L % 4 == 2, L < 1024 (t0 + 1 < L predicates)           | the C ABI's L                  | test_window_abi_lengths           |
| out_start on tile edges and their halo, column-row and span   | out_start                      | test_window_sweep (win_starts)    |
| edges, pass-3 register slot groups (2048 NB R2), both ends,   |                                |                                   |
| odd and even                                                  |                                |                                   |
| row_start > 0 with out_start <, = and > row_start             | the tables                     | test_window_sweep, test_window_abi_lengths |
| no window stores its context (no race between windows)       | overlapping windows, one set   | test_window_sweep (sentinel, one launch per window) |
| out_start < 0, = L - 1, >= L                                  | out_start                      | test_window_out_of_range_out_start |
| contents before row_start: zeros, random, NaN, +-inf          | the caller's buffer            | test_window_context_contents, test_window_abi_lengths |
| channel groups (c0 > 0, ragged last group)                    | workspace size                 | test_window_channel_groups        |
| a set of more than 65,535 windows (ops._window_launches)      | number of windows              | test_window_split_set             |
| 64-bit offsets (seg_base + c total past 2^31)                 | C total                        | test_window_64bit_offsets         |

The 33 window-mode instantiations (three modes x LOGM1 = 0..10) and COL_GATE_PACKED reached through
core_fwd_windows are the ("core" | "plain", LOGM1, L%4==0) cells of test_window_sweep; test_coverage_table asserts them
with the edge cells.  Outputs are held to 1e-3 rel with the absolute term scaled by max|ref| (tests/parity_util.py),
against the fp32 twin and the fp64 truth.  The tests marked ``gpu`` need an H100; the reference self-checks, the
planted-bug rejections and the coverage table run on the CPU.
"""
import math
import os
import re
from importlib import import_module

import pytest
import torch

from tests import parity_util as PU
from tests.test_gpu_fft_core_paths import _act, core_ref, decaying_filter
from tests.test_gpu_packed_core_paths import ABI_L, SENTINEL, _bits, _kpad, _sentinel, abi_starts, packed_starts
from tests.test_gpu_ragged import _exact_workspace
from tests.test_gpu_rows_core_paths import fftconv_pow2, masked_geometry
from tests.test_gpu_widths import NANS, _poison
from tests.test_stream_cpu import causal_conv, direct_core, windowed_core

ops = import_module("hyena_dna_b200.ops")
gpu = pytest.mark.gpu
ROUTES = ("core", "plain")


# ------------------------------------------------------------------------------------------ geometry
def window_epilogue_slots():
    """Slots the window modes' pass 3 keeps in flight: NB of the register-path loop in csrc/fft_passes.cuh, the default
    of its expression (the window modes never run the staged epilogue)."""
    with open(os.path.join(ops._lib.CSRC, "fft_passes.cuh")) as f:
        m = re.search(r"constexpr int NB = (.*\(MODE == INV_BWD_DG_PACKED\) \? \d+ : (\d+));", f.read())
    assert m and "_WIN" not in m.group(1), "the window modes' slot count is no longer where this test reads it"
    return int(m.group(2))


def window_geometry(L):
    """masked_geometry(L) plus the edges of the register-path slot groups of pass 3: on the TWO sizes slot s holds the
    column-FFT rows R2 s .. R2 s + R2 - 1, so a group of NB slots covers 2048 NB R2 samples."""
    g = masked_geometry(L)
    w = 2048 * window_epilogue_slots() * g["r2"]
    g["boundaries"]["slot_group"] = list(range(w, L, w)) if g["two"] else []
    return g


def win_starts(L):
    """out_start values of the sweep: packed_starts(L) (tile edges and their halo, column-row, staged-batch and span
    edges, the ends), the first and last slot-group edge +-2, 0, 1, L / 2, L / 2 + 1, L - 2 and L - 1.  Past L = 2^17
    every window's host reference costs a whole row, so one value of each kind stands for the rest."""
    b = window_geometry(L)["boundaries"]
    sg = b["slot_group"]
    if L > 1 << 17:
        s = {0, 1, 2, L // 2, L // 2 + 1, L - 3, L - 2, L - 1, b["row"][0] - 1, b["row"][-1], b["row"][-1] + 1,
             b["span"][0], b["span"][-1] + 1}
        s |= {e + d for e in (b["tile"][0], sg[0]) for d in range(-2, 3)}
    else:
        s = set(packed_starts(L)) | {0, 1, L // 2, L // 2 + 1, L - 2, L - 1}
        s |= {e + d for e in sg[:1] + sg[-1:] for d in range(-2, 3)}
    return sorted(v for v in s if 0 <= v < L)


def rs_picks(L):
    """row_start values of the sweep's windows with rs > 0: 3, the first tile edge + 1 and the first slot-group edge - 1
    (where they exist), and L / 2 + 1."""
    b = window_geometry(L)["boundaries"]
    s = {3, L // 2 + 1} | ({b["tile"][0] + 1} if b["tile"] else set()) | \
        ({b["slot_group"][0] - 1} if b["slot_group"] else set())
    return sorted(s)


def tile_windows(L, pairs, seed):
    """Overlapping windows of L positions, one per (row_start, out_start) pair in a seeded order, whose stored ranges
    [seg_base + e, seg_base + L) (e = max(os, rs)) tile [head, T - 5) back to back: each window's context is the previous
    windows' stored positions.  head = max(e - rs) + 3 positions are only read, so seg_base + rs >= 0 for every window.
    -> (wins [(seg_base, rs, os)], T)."""
    g = torch.Generator().manual_seed(seed)
    pairs = [pairs[i] for i in torch.randperm(len(pairs), generator=g).tolist()]
    pos = max(max(o, r) - r for r, o in pairs) + 3
    wins = []
    for r, o in pairs:
        e = max(o, r)
        wins.append((pos - e, r, o))
        pos += L - e
    return wins, pos + 5


def sweep_windows(L, seed=0):
    """The sweep's windows at L_b = L: row_start 0 with out_start on every win_starts(L), and for each r of rs_picks(L)
    three windows with row_start r and out_start r - 3, r and r + 3."""
    pairs = [(0, v) for v in win_starts(L)] + [(r, r + d) for r in rs_picks(L) for d in (-3, 0, 3)]
    return tile_windows(L, pairs, seed)


def gap_windows(L, pairs, seed):
    """Windows of L positions that share no position: window j owns [seg_base, seg_base + L), with gaps of 1 to 4
    positions between, before and after; listed in a seeded order.  -> (wins, T)."""
    g = torch.Generator().manual_seed(seed)
    wins, a = [], 0
    for r, o in pairs:
        a += 1 + int(torch.randint(0, 4, (1,), generator=g))
        wins.append((a, r, o))
        a += L
    T = a + 1 + int(torch.randint(0, 4, (1,), generator=g))
    return [wins[i] for i in torch.randperm(len(wins), generator=g).tolist()], T


def abi_pairs(L):
    """(row_start, out_start) of the C ABI cases: on abi_starts(L) e, in turn (e, e), (e - 1000 or 0, e) (context
    read) and (e, e - 2) (out_start < row_start)."""
    out = []
    for j, e in enumerate(abi_starts(L)):
        out.append([(e, e), (max(0, e - 1000), e), (e, e - 2)][j % 3])
    return out


def stored_mask(wins, L, T):
    m = torch.zeros(T, dtype=torch.bool)
    for sg, r, o in wins:
        e = max(o, r)
        if e < L:
            m[sg + e:sg + L] = True
    return m


def read_mask(wins, L, T):
    """Positions some window reads: [seg_base + rs, seg_base + L)."""
    m = torch.zeros(T, dtype=torch.bool)
    for sg, r, _ in wins:
        m[max(0, sg + r):sg + L] = True
    return m


def _tables(wins, dev):
    return (torch.tensor([w[0] for w in wins], dtype=torch.int64, device=dev),
            torch.tensor([w[1] for w in wins], dtype=torch.int32, device=dev),
            torch.tensor([w[2] for w in wins], dtype=torch.int32, device=dev))


# ------------------------------------------------------------------------------------------ per-window fp64 reference
PLANTED = ["context stored", "os+1", "os-1", "max(os, rs) dropped", "read before row_start", "seg_base+1",
           "Dvec dropped"]


def window_ref(x, wins, L, t, route, dtype=torch.float64, bug=None):
    """The windows on the host, each alone: route "core" runs core_ref on p[..., seg_base + rs : seg_base + L] (x = p (1,
    3D, T)) with k cut to L - rs, route "plain" fftconv_pow2 on u's slice (x = u (1, H, T)) with the D skip term.
    Returns (y (1, C, T), written (T,) bool): each window's outputs at [seg_base + e, seg_base + L), e = max(os, rs), in
    the windows' order (a later window overwrites an earlier one, as a launch that writes out of turn would).

    ``bug`` plants one error: "context stored" (e = rs), "os+1" / "os-1" (out_start off by one), "max(os, rs) dropped"
    (stores from max(os, 0): the outputs before rs, which read only zeros, are 0), "read before row_start" (every window
    reads from rs - 1), "seg_base+1" (every window addressed one position late), "Dvec dropped" (the plain route
    without its skip term)."""
    C = x.shape[1] // 3 if route == "core" else x.shape[1]
    T = x.shape[-1]
    k = _kpad(t["k"], L)
    y = torch.zeros(1, C, T, dtype=dtype)
    written = torch.zeros(T, dtype=torch.bool)
    plan = []
    for sg, r, o in wins:
        sg += bug == "seg_base+1"
        lo = r - 1 if bug == "read before row_start" else r
        e = {"context stored": r, "os+1": max(o + 1, r), "os-1": max(o - 1, r),
             "max(os, rs) dropped": max(o, 0)}.get(bug, max(o, r))
        plan.append((sg, lo, e))
    by_lo = {}
    for i, (sg, lo, e) in enumerate(plan):
        if e < L:
            by_lo.setdefault(lo, []).append(i)
    got = {}
    for lo, idx in by_lo.items():
        n = L - lo
        step = max(1, (1 << 21) // L)
        for j in range(0, len(idx), step):
            part = idx[j:j + step]
            xs = torch.cat([x[:, :, plan[i][0] + lo:plan[i][0] + L] for i in part])
            if route == "core":
                r = core_ref(xs, t["ib"], t["sw"], t["sb"], k[:, :n], t["fb"], torch.zeros(len(part), C, n),
                             dtype=dtype, conv=fftconv_pow2)["y"]
            else:
                Dv = torch.zeros_like(t["Dv"]) if bug == "Dvec dropped" else t["Dv"]
                r = fftconv_pow2(xs.to(dtype), k[:, :n].to(dtype), Dv.to(dtype))
            for m, i in enumerate(part):
                e = plan[i][2]
                got[i] = r[m, :, max(e, lo) - lo:].clone()
    for i in sorted(got):
        sg, lo, e = plan[i]
        y[0, :, sg + e:sg + max(e, lo)] = 0.0             # positions before rs: their outputs read only zeros
        y[0, :, sg + max(e, lo):sg + L] = got[i]
        written[sg + e:sg + L] = True
    return y, written


def window_refs(x, wins, L, t, route):
    """(fp32 reference, fp64 truth) of window_ref."""
    return window_ref(x, wins, L, t, route, torch.float32)[0], window_ref(x, wins, L, t, route, torch.float64)[0]


def planted_output(x, wins, L, t, route, bug):
    """What a kernel with ``bug`` leaves in a SENTINEL-filled fp32 output."""
    y, written = window_ref(x, wins, L, t, route, bug=bug)
    o = torch.full(y.shape, SENTINEL, dtype=torch.int32).view(torch.float32)
    o[..., written] = y[..., written].float()
    return o


def check_windows(o, r32, r64, wins, L, tag):
    """Every position no window stores keeps the sentinel's bits; every stored one is held to the truth."""
    st = stored_mask(wins, L, o.shape[-1])
    assert bool((_bits(o)[..., ~st] == SENTINEL).all()), f"{tag}: written outside the windows' stored ranges"
    _act(o[..., st], r32[..., st], r64[..., st], tag)


# ------------------------------------------------------------------------------------------ inputs
def window_inputs(route, D, T, L, seed, big=None, fill_mask=None, fill=None):
    """Seeded host inputs: p (1, 3D, T) with the core's parameters, or u (1, D, T) with Dv; a decaying filter k (D, L).
    Positions in ``big`` hold values of magnitude 3 to 10; positions in ``fill_mask`` hold ``fill`` ("zero", an int
    seed for large random values, a NaN encoding of tests/test_gpu_widths.NANS or "inf")."""
    g = torch.Generator().manual_seed(seed)
    name = "p" if route == "core" else "u"
    x = torch.randn(1, 3 * D if route == "core" else D, T, generator=g)
    t = dict(k=decaying_filter(D, L, g))
    if route == "core":
        t.update(ib=torch.randn(3 * D, generator=g) * 0.5, sw=(torch.rand(3 * D, 3, generator=g) * 2 - 1) / math.sqrt(3),
                 sb=(torch.rand(3 * D, generator=g) * 2 - 1) / math.sqrt(3), fb=torch.randn(D, generator=g))
    else:
        t.update(Dv=torch.randn(D, generator=g))
    if big is not None:
        n = int(big.sum())
        x[..., big] = (3 + 7 * torch.rand(x.shape[1], n, generator=g)) * torch.randn(x.shape[1], n, generator=g).sign()
    if fill_mask is not None:
        if fill == "zero":
            v = torch.zeros_like(x)
        elif isinstance(fill, int):
            gs = torch.Generator().manual_seed(fill)
            v = (3 + 7 * torch.rand(x.shape, generator=gs)) * torch.randn(x.shape, generator=gs).sign()
        else:
            v = _poison(x, fill, g)
        x = torch.where(fill_mask, v, x)
    t[name] = x
    return t


def context_mask(wins, L, T):
    """Positions that are some window's context: [seg_base + rs, seg_base + max(os, rs))."""
    m = torch.zeros(T, dtype=torch.bool)
    for sg, r, o in wins:
        m[sg + r:sg + min(L, max(o, r))] = True
    return m


def _x(t, route):
    return t["p"] if route == "core" else t["u"]


# ------------------------------------------------------------------------------------------ sweep and coverage table
SWEEP_LB = [1 << e for e in range(10, 21)]


def decisions_sweep(L):
    """Cells of the coverage table the sweep's windows at L_b = L reach (both routes run the same windows)."""
    g = window_geometry(L)
    b, m = g["boundaries"], g["logm1"]
    wins, _ = sweep_windows(L)
    os_ = {o for _, r, o in wins if r == 0}
    out = {(r, m, "L%4==0") for r in ROUTES} | {("COL_GATE_PACKED", m)}
    if g["two"] and all(b["tile"][0] + d in os_ for d in range(-2, 3)):
        out.add(("tile halo", m))
    if any(e in os_ for e in b["row"]):
        out.add(("column-row edge", m))
    if any(e in os_ for e in b["span"]):
        out.add(("span edge", m))
    if b["slot_group"] and all(b["slot_group"][0] + d in os_ for d in range(-2, 3)):
        out.add(("slot-group edge", m))
    if {0, L - 1} <= os_:
        out.add(("both ends", m))
    if {o % 2 for o in os_ if 2 < o < L - 2} == {0, 1}:
        out.add(("odd and even out_start", m))
    if {"<" if o < r else "=" if o == r else ">" for _, r, o in wins if r > 0} == {"<", "=", ">"}:
        out.add(("row_start > 0, out_start <, =, >", m))
    return out


def decisions_abi(L):
    m = masked_geometry(L)["logm1"]
    kind = "L%4==0" if L % 4 == 0 else ("odd" if L % 2 else "L%4==2")
    return {(r, m, kind) for r in ROUTES} | ({("L < 1024",)} if L < 1024 else set())


def test_coverage_table():
    """The sweep and the C ABI cases reach every LOGM1 through both entry points with L % 4 == 0 and odd L; at every
    LOGM1 out_start at both ends and on odd and even values, windows with row_start > 0 and out_start below, at and past
    it; on the TWO sizes the first tile edge's halo and the first slot-group edge +-2; column-row and span edges wherever
    the row has them."""
    hit = set()
    for L in SWEEP_LB:
        hit |= decisions_sweep(L)
    for L in ABI_L:
        hit |= decisions_abi(L)
    want = {(r, m, kind) for r in ROUTES for m in range(11) for kind in ("L%4==0", "odd")}
    want |= {("COL_GATE_PACKED", m) for m in range(11)} | {("L < 1024",)}
    want |= {(cell, m) for cell in ("both ends", "odd and even out_start", "row_start > 0, out_start <, =, >")
             for m in range(11)}
    want |= {(cell, m) for cell in ("tile halo", "slot-group edge") for m in range(5, 11)}
    want |= {("column-row edge", m) for m in range(2, 11)} | {("span edge", m) for m in range(4, 11)}
    assert not want - hit, f"table cells not hit: {sorted(want - hit, key=str)}"
    # the geometry the cells rest on: four slots per register-path group, so 2048 * 4 * 32 samples at 2^20
    assert window_epilogue_slots() == 4
    assert window_geometry(1 << 20)["boundaries"]["slot_group"] == [262144, 524288, 786432]
    assert window_geometry(1 << 15)["boundaries"]["slot_group"] == [8192, 16384, 24576]
    for L in SWEEP_LB:                         # the layout's promises: disjoint stored ranges that tile [head, T - 5)
        wins, T = sweep_windows(L)
        hits = torch.zeros(T, dtype=torch.int64)
        for sg, r, o in wins:
            assert sg + r >= 0 and sg + L <= T and 0 <= r < L
            hits[sg + max(o, r):sg + L] += 1
        head = max(max(o, r) - r for _, r, o in wins) + 3
        assert bool((hits[head:T - 5] == 1).all()) and not bool(hits[:head].any()) and not bool(hits[T - 5:].any())
    for L in ABI_L:
        wins, T = gap_windows(L, abi_pairs(L), L)
        assert all(sg >= 1 and sg + L < T for sg, _, _ in wins)


# ------------------------------------------------------------------------------------------ CPU self-checks
def test_window_ref_is_the_stream_model_and_the_direct_convolution():
    """window_ref on the windows of ops.stream_windows (one row, one channel) is tests/test_stream_cpu.windowed_core and,
    with enough context, direct_core over the whole row; the plain route is the whole row's causal convolution with its
    D skip term.  Both with the windows in a shuffled order and their stored ranges disjoint."""
    g = torch.Generator().manual_seed(3)
    n, L, l_max = 3000, 1024, 61
    p = torch.randn(3, n, generator=g, dtype=torch.float64)
    k = torch.randn(l_max, generator=g, dtype=torch.float64)
    bias = torch.randn(1, generator=g, dtype=torch.float64)[0]
    sw = torch.randn(3, 3, generator=g, dtype=torch.float64)
    sb = torch.randn(3, generator=g, dtype=torch.float64)
    wins = ops.stream_windows(n, L, ops.stream_context(l_max, 2))
    t = dict(ib=torch.zeros(3, dtype=torch.float64), sw=sw, sb=sb, k=k[None], fb=bias.reshape(1))
    y, written = window_ref(p[None], wins[::-1], L, t, "core")
    assert bool(written.all())
    torch.testing.assert_close(y[0, 0], windowed_core(p, k, bias, sw, sb, wins, L), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(y[0, 0], direct_core(p, k, bias, sw, sb), rtol=1e-9, atol=1e-9)
    u = torch.randn(1, 2, n, generator=g, dtype=torch.float64)
    kk = torch.randn(2, l_max, generator=g, dtype=torch.float64)
    Dv = torch.randn(2, generator=g, dtype=torch.float64)
    wins = ops.stream_windows(n, L, ops.stream_context(l_max, 1))
    y, written = window_ref(u, wins, L, dict(k=kk, Dv=Dv), "plain")
    assert bool(written.all())
    torch.testing.assert_close(y, causal_conv(u, kk, Dv), rtol=1e-9, atol=1e-9)


def _small_case(route, seed=5):
    """Windows of L_b = 64 over one buffer (D = 3): row_start 0 with out_start 0, 1, 2, 31, 62, 63, and row_start 5
    with out_start 2, 5 and 9, their context large."""
    L = 64
    pairs = [(0, v) for v in (0, 1, 2, 31, 62, 63)] + [(5, 2), (5, 5), (5, 9)]
    wins, T = tile_windows(L, pairs, seed)
    t = window_inputs(route, 3, T, L, seed, big=context_mask(wins, L, T))
    return wins, T, L, t


@pytest.mark.parametrize("route,bug", [(r, b) for r in ROUTES for b in PLANTED if b != "Dvec dropped" or r == "plain"])
def test_parity_bar_rejects_planted_window_bugs(route, bug):
    """Each planted window bug is rejected by the bar (check_windows: the sentinel outside the stored ranges, the
    tolerance inside) that the unplanted reference passes."""
    wins, T, L, t = _small_case(route)
    x = _x(t, route)
    r32, r64 = window_refs(x, wins, L, t, route)
    n0 = len(PU._records)
    try:
        check_windows(planted_output(x, wins, L, t, route, None), r32, r64, wins, L, "unplanted")
        with pytest.raises(AssertionError):
            check_windows(planted_output(x, wins, L, t, route, bug), r32, r64, wins, L, f"planted {bug}")
    finally:
        del PU._records[n0:]            # self-checks of the bar, not parity records


# ------------------------------------------------------------------------------------------ device helpers
def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _params(t, route, dev):
    return {n: t[n].to(dev) for n in (("ib", "sw", "sb", "fb") if route == "core" else ("Dv",))}


def windows_run(H, t, wins, L, dev, route, one_at_a_time=False, on_device=False):
    """The window entry point of ``route`` as ops.core_forward_windows / fftconv_forward_windows call it (kspec of
    ops._bucket_filter(k, L_b), ops.workspace, one launch per 65,535 windows), into a caller-owned output pre-filled
    with SENTINEL; ``one_at_a_time``: one launch per window, in the tables' order, into the same output."""
    lib, P = H._lib.lib(), ops._ptr
    x = _x(t, route) if on_device else _x(t, route).to(dev)
    _, Cx, T = x.shape
    C = Cx // 3 if route == "core" else Cx
    kspec = ops.filter_spectrum(ops._bucket_filter(t["k"].to(dev), L))
    q = _params(t, route, dev)
    sg, rs, os_ = _tables(wins, dev)
    out = _sentinel((1, C, T), dev)
    sets = [(i, 1) for i in range(len(wins))] if one_at_a_time else list(ops._window_launches(len(wins)))
    for r0, n in sets:
        ws = ops.workspace(n, C, L, False, dev)
        if route == "core":
            H._lib.check(lib.hyena_b200_core_fwd_windows(
                P(x), P(q["ib"]), P(q["sw"]), P(q["sb"]), P(kspec), P(q["fb"]), P(out), P(sg[r0:]), P(rs[r0:]),
                P(os_[r0:]), T, n, C, L, P(ws), ws.numel(), ops._stream()))
        else:
            H._lib.check(lib.hyena_b200_fftconv_fwd_windows(
                P(x), P(kspec), P(q["Dv"]), P(out), P(sg[r0:]), P(rs[r0:]), P(os_[r0:]), T, n, C, L, P(ws),
                ws.numel(), ops._stream()))
    torch.cuda.synchronize()
    return out if on_device else out.cpu()


def ops_windows_run(t, wins, L, dev, route):
    """ops.core_forward_windows / ops.fftconv_forward_windows on the same windows (positions no window stores are
    undefined there)."""
    x = _x(t, route).to(dev)
    kspec = ops.filter_spectrum(ops._bucket_filter(t["k"].to(dev), L))
    q = _params(t, route, dev)
    tables = _tables(wins, dev)
    if route == "core":
        y = ops.core_forward_windows(x, q["ib"], q["sw"], q["sb"], kspec, q["fb"], L, tables)
    else:
        y = ops.fftconv_forward_windows(x, kspec, q["Dv"], L, tables)
    torch.cuda.synchronize()
    return y.cpu()


def run_and_check(H, dev, t, wins, L, route, tag, refs=None):
    x = _x(t, route)
    r32, r64 = refs or window_refs(x, wins, L, t, route)
    o = windows_run(H, t, wins, L, dev, route)
    check_windows(o, r32, r64, wins, L, tag)
    return o, (r32, r64)


# ------------------------------------------------------------------------------------------ 1. transform size sweep
@gpu
@pytest.mark.parametrize("L", SWEEP_LB)
@pytest.mark.parametrize("route", ROUTES)
def test_window_sweep(route, L):
    """Overlapping windows of L_b = L over one buffer (D = 2) whose stored ranges tile it, with out_start on every
    win_starts(L) and row_start > 0 with out_start below, at and past it, their context large: every stored position
    against the truth, every other one keeps the sentinel's bits, and the whole buffer is bit for bit that of the same
    windows launched one at a time (no window writes another's positions, whatever the order).  ops' route gives the
    same bits at every stored position."""
    H = _H()
    dev = _dev()
    wins, T = sweep_windows(L, seed=L)
    t = window_inputs(route, 2, T, L, seed=L + 1, big=context_mask(wins, L, T))
    o, _ = run_and_check(H, dev, t, wins, L, route, f"window sweep {route} L_b={L} windows={len(wins)}")
    one = windows_run(H, t, wins, L, dev, route, one_at_a_time=True)
    assert torch.equal(_bits(one), _bits(o)), f"{route} L_b={L}: the set differs from one launch per window"
    st = stored_mask(wins, L, T)
    via = ops_windows_run(t, wins, L, dev, route)
    assert torch.equal(_bits(via[..., st]), _bits(o[..., st])), f"{route} L_b={L}: ops route differs"


# ------------------------------------------------------------------------------------------ 2. the C ABI contract
@gpu
@pytest.mark.parametrize("L", ABI_L)
@pytest.mark.parametrize("route", ROUTES)
def test_window_abi_lengths(route, L):
    """Any L through the C entry points, windows that share no position (abi_pairs: out_start on abi_starts, context
    read, out_start < row_start), whose positions before row_start and the gaps hold NaN or +-inf: every position no
    window stores keeps the sentinel's bits, everything stored is within the bar."""
    H = _H()
    dev = _dev()
    wins, T = gap_windows(L, abi_pairs(L), seed=L)
    fill = [*NANS, "inf"][L % 4]
    t = window_inputs(route, 2, T, L, seed=3 * L + 1, fill_mask=~read_mask(wins, L, T), fill=fill)
    run_and_check(H, dev, t, wins, L, route, f"window abi {route} L={L} pre-rs {fill}")


# ------------------------------------------------------------------------------------------ 3. out_start out of range
@gpu
@pytest.mark.parametrize("L", [1024, 32767])
@pytest.mark.parametrize("route", ROUTES)
def test_window_out_of_range_out_start(route, L):
    """out_start < 0 stores from row_start, out_start = L - 1 stores one position, out_start >= L (up to 2^31 - 1)
    stores nothing: against the truth with the sentinel elsewhere, and a set of only the last kind leaves the output all
    sentinel."""
    H = _H()
    dev = _dev()
    none = [(0, L), (3, L + 1), (0, 2 ** 31 - 1)]
    pairs = [(5, -7), (0, -1), (0, -(2 ** 31)), (3, L - 1), (0, L - 1), (7, 8)] + none
    wins, T = gap_windows(L, pairs, seed=L + 11)
    t = window_inputs(route, 2, T, L, seed=L + 12, fill_mask=~read_mask(wins, L, T), fill="inf")
    run_and_check(H, dev, t, wins, L, route, f"window out_start range {route} L={L}")
    assert int(stored_mask([w for w in wins if (w[1], w[2]) in [(3, L - 1), (0, L - 1)]], L, T).sum()) == 2
    o = windows_run(H, t, [w for w in wins if (w[1], w[2]) in none], L, dev, route)
    assert bool((_bits(o) == SENTINEL).all()), f"{route} L={L}: a window with out_start >= L stored something"


# ------------------------------------------------------------------------------------------ 4. contents before rs
@gpu
@pytest.mark.parametrize("L", [1 << 15, 1 << 20])
@pytest.mark.parametrize("route", ROUTES)
def test_window_context_contents(route, L):
    """Windows with row_start 1, 2, 3, 2047, L / 2 + 1 and L - 5, their positions before row_start (and the gaps)
    holding zeros, random values, the NaN encodings and +-inf: every stored output keeps its bits; with zeros, against
    the truth."""
    H = _H()
    dev = _dev()
    pairs = [(r, r + j % 3) for j, r in enumerate((1, 2, 3, 2047, L // 2 + 1, L - 5))]
    wins, T = gap_windows(L, pairs, seed=L + 21)
    outside = ~read_mask(wins, L, T)
    st = stored_mask(wins, L, T)
    zero, _ = run_and_check(H, dev, window_inputs(route, 2, T, L, 97, fill_mask=outside, fill="zero"), wins, L, route,
                            f"window contents zero {route} L_b={L}")
    for fill in (1, 2, *NANS, "inf"):
        o = windows_run(H, window_inputs(route, 2, T, L, 97, fill_mask=outside, fill=fill), wins, L, dev, route)
        assert torch.equal(_bits(o[..., st]), _bits(zero[..., st])), f"{route} L_b={L} {fill}: stored outputs changed"
        assert bool((_bits(o[..., ~st]) == SENTINEL).all()), f"{route} L_b={L} {fill}: written outside"


# ------------------------------------------------------------------------------------------ 5. channel groups
KINDS = {"core": ("col_fwd<gate>", "row_pass<conv_fwd>", "col_inv<conv_fwd>"),
         "plain": ("col_fwd<plain>", "row_pass<conv_fwd>", "col_inv<plain_fwd>")}


@gpu
@pytest.mark.parametrize("route", ROUTES)
def test_window_channel_groups(monkeypatch, route):
    """The workspace cut to 3 channels per launch (D = 7: 3 + 3 + 1, c0 > 0, a ragged last group) on the sweep's
    windows at L_b = 4096: against the truth, three launches per pass, and bit for bit the one-group run."""
    H = _H()
    dev = _dev()
    L = 4096
    wins, T = sweep_windows(L, seed=7)
    t = window_inputs(route, 7, T, L, seed=59, big=context_mask(wins, L, T))
    H._lib.profile_begin()
    base, refs = run_and_check(H, dev, t, wins, L, route, f"window groups {route} one group")
    prof = H._lib.profile_end()
    assert all(prof[k][1] == 1 for k in KINDS[route]), prof
    monkeypatch.setattr(ops, "workspace", _exact_workspace(H, 3))
    H._lib.profile_begin()
    got, _ = run_and_check(H, dev, t, wins, L, route, f"window groups {route} G=3", refs=refs)
    prof = H._lib.profile_end()
    assert all(prof[k][1] == 3 for k in KINDS[route]), prof
    assert torch.equal(_bits(got), _bits(base)), f"window groups {route}: differs from the one-group run"


# ------------------------------------------------------------------------------------------ 6. split window sets
def _direct_last(x, t, route, L, i0, i1, dtype):
    """Output at window position L - 1 of windows i = i0 .. i1 - 1 at seg_base i, row_start 0, by direct sums: the
    short filter on the window (zeros before it), then sum_j k[j] g[L - 1 - j] + fb g[L - 1] (core), or
    sum_j k[j] u[L - 1 - j] + D u[L - 1] (plain)."""
    w = x[0].to(dtype).unfold(1, L, 1)[:, i0:i1].transpose(0, 1)                 # (n, C, L)
    k = t["k"].to(dtype)[:, :L].flip(-1)
    if route == "plain":
        return (w * k).sum(-1) + t["Dv"].to(dtype) * w[..., -1]
    C3 = w.shape[1]
    D = C3 // 3
    s = torch.nn.functional.conv1d(w + t["ib"].to(dtype)[None, :, None], t["sw"].to(dtype)[:, None, :],
                                   t["sb"].to(dtype), padding=2, groups=C3)[..., :L]
    x0, x1, v = s.split(D, dim=1)
    g = x1 * v
    return ((g * k).sum(-1) + t["fb"].to(dtype) * g[..., -1]) * x0[..., -1]


@gpu
@pytest.mark.parametrize("route", ROUTES)
def test_window_split_set(route):
    """65,535 + 5 windows of L_b = 1024 at seg_base i, each storing its last position (out_start 1023), over a buffer of
    66,563 positions, D = 1, through ops.core_forward_windows / fftconv_forward_windows: two launches per pass, the second
    reading its tables at 65,535, every output against its direct sum."""
    H = _H()
    dev = _dev()
    L, N = 1024, ops.MAX_BUCKET_ROWS + 5
    T = N + L + 4
    wins = [(i, 0, L - 1) for i in range(N)]
    t = window_inputs(route, 1, T, L, seed=67)
    x = _x(t, route)
    kspec = ops.filter_spectrum(ops._bucket_filter(t["k"].to(dev), L))
    q = _params(t, route, dev)
    tables = _tables(wins, dev)
    xd = x.to(dev)
    H._lib.profile_begin()
    if route == "core":
        y = ops.core_forward_windows(xd, q["ib"], q["sw"], q["sb"], kspec, q["fb"], L, tables)
    else:
        y = ops.fftconv_forward_windows(xd, kspec, q["Dv"], L, tables)
    prof = H._lib.profile_end()
    assert all(prof[k][1] == 2 for k in KINDS[route]), prof
    got = y.cpu()[0, :, L - 1:L - 1 + N]
    refs = [torch.cat([_direct_last(x, t, route, L, i0, min(N, i0 + 8192), dt) for i0 in range(0, N, 8192)]).T
            for dt in (torch.float32, torch.float64)]
    _act(got, refs[0], refs[1], f"window split set {route} {N} windows")


# ------------------------------------------------------------------------------------------ 7. 64-bit offsets
@gpu
@pytest.mark.parametrize("route", ROUTES)
def test_window_64bit_offsets(route):
    """Windows of L_b = 2^20 at the end of a buffer whose channel offsets pass 2^31.  Core: D = 256 and T = 3,146,724,
    so the v rows (2D + c) T of channels c >= 170 lie past element 2^31 at these windows (169 below): channels 0, 169,
    170, 171 and 255.  Plain: u (1, 2, 2^30 + 2^20), channel 1's windows past 2^31, one straddling it: both channels.
    Each against the truth of those channels alone (both routes are depthwise)."""
    H = _H()
    dev = _dev()
    L = 1 << 20
    if route == "core":
        D, T, chans = 256, 3146724, [0, 169, 170, 171, 255]
        wins = [(T - L, 0, L - 3000), (T - 3000 - L, 0, L - 5000), (T - 8000 - L, 1 << 19, L - 2000)]
        assert (2 * D + 170) * T <= 2 ** 31 <= (2 * D + 170) * T + min(sg + r for sg, r, _ in wins)
    else:
        D, T, chans = 2, (1 << 30) + (1 << 20), [0, 1]
        wins = [(T - L, 0, 1 << 19), (T - (1 << 19) - L, 0, 0), (T - 3 * (1 << 19) - L, 1000, (1 << 18) + 1)]
        lo = T - 3 * (1 << 19) - L + (1 << 18) + 1
        assert T + lo < 2 ** 31 < T + T - 3 * (1 << 19)
    g = torch.Generator(device=dev).manual_seed(71)
    gh = torch.Generator().manual_seed(72)
    a = min(sg + r for sg, r, _ in wins)                  # the first position any window reads
    t = dict(k=decaying_filter(D, L, gh))
    if route == "core":
        t.update(p=torch.randn(1, 3 * D, T, generator=g, device=dev), ib=torch.randn(3 * D, generator=gh) * 0.5,
                 sw=(torch.rand(3 * D, 3, generator=gh) * 2 - 1) / math.sqrt(3),
                 sb=(torch.rand(3 * D, generator=gh) * 2 - 1) / math.sqrt(3), fb=torch.randn(D, generator=gh))
        rows = [c + j * D for j in range(3) for c in chans]
    else:
        t.update(u=torch.randn(1, D, T, generator=g, device=dev), Dv=torch.randn(D, generator=gh))
        rows = chans
    try:
        o = windows_run(H, t, wins, L, dev, route, on_device=True)
        got = o[:, chans, a:].cpu()
        untouched = bool((o[:, :, :a].view(torch.int32) == SENTINEL).all())
        x = _x(t, route)[:, rows, a:].cpu()
    finally:
        t["p" if route == "core" else "u"] = o = None
        ops._ws_cache.clear()
        torch.cuda.empty_cache()
    assert untouched, f"window 64-bit {route}: written before the windows"
    sub = dict(t, k=t["k"][chans])
    if route == "core":
        sub.update(ib=t["ib"][rows], sw=t["sw"][rows], sb=t["sb"][rows], fb=t["fb"][chans])
    else:
        sub.update(Dv=t["Dv"][chans])
    local = [(sg - a, r, os_) for sg, r, os_ in wins]
    r32, r64 = window_refs(x, local, L, sub, route)
    check_windows(got, r32, r64, local, L, f"window 64-bit {route} channels {chans}")
