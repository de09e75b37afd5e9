"""The order-2 FFT core on packed sequences against fp64: the packed modes at every transform size.

``hyena_b200_core_fwd_packed`` / ``core_bwd_packed`` / ``short_bwd_packed`` (DESIGN.md section 4.18) run COL_GATE_PACKED
and INV_CONV_FWD_PACKED forward, COL_DC_PACKED, INV_BWD_DG_PACKED (and COL_GATE_PACKED without a saved g spectrum)
backward, and short_conv_bwd_packed_kernel for dp and d in_proj.bias, once per bucket of rows of one length L_b.  Row b
of a bucket reads and writes the packed tensors at seg_base[b] + t for t in [row_start[b], L_b) only.  The tests drive
the three entry points directly (``packed_run``, which mirrors ops.core_forward_packed / core_backward_packed but owns
its output buffers, so ds is visible and untouched positions can be checked), with the plan of ops.packed_plan or with
hand-made seg_base / row_start tables (the C ABI accepts any L <= 2^20, any row start and any layout).

Truth is per sequence: sequence i alone is the *_ROWS problem on its slice, so ``packed_core_ref`` runs the fp64 core
(tests/test_gpu_fft_core_paths.core_ref, as tests/test_gpu_rows_core_paths.rows_core_ref does per row) on the slices of
each length at once, with its fp32 twin; parameter gradients are the sums over the sequences and dk the sum of each
bucket's dk cut to min(L_b, Lk).

| decision                                                   | selected by                       | test                               |
|------------------------------------------------------------|-----------------------------------|------------------------------------|
| transform template LOGM1 = 0..10, L % 4 == 0               | bucket length L_b                 | test_packed_core_sweep             |
| odd L, L % 4 == 2, L < 1024 (t0 + 1 < L predicates)        | the C ABI's L                     | test_abi_lengths                   |
| row_start on tile edges and their halo, column-row edges,  | row_start = L_b - n               | test_packed_core_sweep (packed_starts), |
| two-slot INV_BWD_DG_PACKED batches, short_conv_bwd spans   |                                   | test_abi_lengths (abi_starts)      |
| buckets launched in either order next to each other        | plan order                        | test_packed_core_sweep             |
| B = 1: ROW_CONV_BWD1 (saved spectrum) / ROW_CONV_BWD       | one row, HYENA_B200_SAVE_SPECTRUM | test_packed_single_row             |
| spectrum recompute (COL_GATE_PACKED in the backward)       | HYENA_B200_SAVE_SPECTRUM=0        | test_packed_single_row             |
| channel groups (c0 > 0, ragged last group)                 | workspace size, 65535 / B         | test_packed_channel_groups, test_packed_natural_group_cut |
| split bucket (bk.offset slices of the device tables)       | > ops.MAX_BUCKET_ROWS sequences   | test_packed_split_bucket           |
| 64-bit packed offsets (v rows wholly past 2^31)            | 3 D total                         | test_packed_64bit_offsets          |
| c_save float2 (vec) / scalar                               | L parity, c_save alignment        | test_abi_lengths, test_abi_c_save_offset |
| nothing outside [row_start, L) read or written             | gaps, seg_base out of cu order    | test_abi_lengths, test_abi_c_save_offset |
| neighbour contents: zeros, random, NaN, +-inf              | the other sequences               | test_packed_neighbour_contents     |
| the packed operator at d_model 1, 2, 3                     | HyenaOperator(cu_seqlens=)        | test_packed_operator_small_widths  |

Activations are held to 1e-3 rel with the absolute term scaled by max|ref| (per bucket), parameter gradients with
``param_grad=True``, both against the fp32 twin of the reference and its fp64 truth (tests/parity_util.py).  The tests
marked ``gpu`` need an H100; the reference self-checks, the planted-bug rejections and the coverage table run on the CPU.
"""
import math
import os
import re
from importlib import import_module

import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_fft_core_paths import _act, _at_offset, _par, core_ref, decaying_filter
from tests.test_gpu_ragged import _exact_workspace
from tests.test_gpu_rows_core_paths import fftconv_pow2, masked_core, masked_geometry, row_starts, rows_core_ref
from tests.test_gpu_widths import NANS, _poison

ops = import_module("hyena_dna_b200.ops")
gpu = pytest.mark.gpu
SENTINEL = 0x7FA5A5A5               # a NaN payload no kernel produces: "this position was never written"


# ------------------------------------------------------------------------------------------ geometry
def packed_epilogue_slots():
    """Slots the packed backward pass 3 keeps in flight: NB of its register-path loop in csrc/fft_passes.cuh."""
    with open(os.path.join(ops._lib.CSRC, "fft_passes.cuh")) as f:
        m = re.search(r"constexpr int NB = .*\(MODE == INV_BWD_DG_PACKED\) \? (\d+) : (\d+);", f.read())
    assert m, "the INV_BWD_DG_PACKED slot count is no longer where this test reads it"
    return int(m.group(1))


def packed_geometry(L):
    """masked_geometry(L) plus the edges of the two-slot batches of INV_BWD_DG_PACKED: on the TWO sizes slot s holds the
    column-FFT rows R2 s .. R2 s + R2 - 1, so a batch of NB slots covers 2048 NB R2 samples."""
    g = masked_geometry(L)
    w = 2048 * packed_epilogue_slots() * g["r2"]
    g["boundaries"]["pair_bwd"] = list(range(w, L, w)) if g["two"] else []
    return g


def packed_starts(L):
    """row_starts(L) (tile edges and their halo, column-row edges, staged-batch edges, short_conv_bwd spans, the ends),
    the first two-slot batch edge of the packed backward +-2 and the first span edge (which row_starts leaves out past
    2^17)."""
    b = packed_geometry(L)["boundaries"]
    s = set(row_starts(L)) | {b["pair_bwd"][0] + d for d in range(-2, 3) if b["pair_bwd"]}
    return sorted(s | set(b["span"][:1]))


def abi_starts(L):
    """Row starts of the C ABI cases: the row's end, the first tile edge's halo, the last tile, column-row and span
    edges +-1, and 0 / 1 while the whole row is affordable on the host.  Sequences stay short past L = 2^16."""
    b = masked_geometry(L)["boundaries"]
    s = {L - 1, L - 2, L - 3, L - 1000, L - 2047}
    for name in ("tile", "row", "span"):
        if b[name]:
            s |= {b[name][-1] + d for d in (-1, 0, 1)}
    if L <= 1 << 16:
        s |= {0, 1} | ({b["tile"][0] + d for d in range(-2, 3)} if b["tile"] else set())
    return sorted(v for v in s if 0 <= v < L)


def seqs_from_cu(cu):
    return [(cu[i], cu[i + 1] - cu[i]) for i in range(len(cu) - 1)]


def _kpad(k, L):
    """k (D, Lk) zero-padded to at least L taps, as ops._bucket_filter pads it."""
    return torch.cat([k, torch.zeros(k.shape[0], max(0, L - k.shape[1]), dtype=k.dtype)], 1)


def make_plan(seqs, rows):
    """PackedBuckets of ``rows`` [(L_b, [sequence indices])] in launch order: seg_base a + n - L_b, row_start L_b - n."""
    plan, off = [], 0
    for L, idx in rows:
        plan.append(ops.PackedBucket(L, list(idx), [seqs[i][0] + seqs[i][1] - L for i in idx],
                                     [L - seqs[i][1] for i in idx], off))
        off += len(idx)
    return plan


# ------------------------------------------------------------------------------------------ per-sequence fp64 reference
def packed_core_ref(p, ib, sw, sb, k, fb, dy, seqs, plan, dtype=torch.float64, conv=fftconv_pow2):
    """core_ref on each sequence's slice alone, the slices of one length in one call (rows_core_ref on the sequence's
    row of its bucket, batched).  p (1, 3D, T) and dy (1, D, T) packed, k (D, Lk), seqs [(offset, n)], plan from
    make_plan / ops.packed_plan.  Returns y (1, D, T), dx (dp) and ds (1, 3D, T), zero outside the sequences; c, one
    (B, D, L_b) per bucket in the row layout (0 at t < row_start); dk (D, Lk), the sum over buckets of each bucket's dk
    cut to min(L_b, Lk); dib, dsw, dsb, dfb summed over the sequences."""
    C3, T = p.shape[1], p.shape[2]
    D, Lk = C3 // 3, k.shape[1]
    z = lambda *s: torch.zeros(*s, dtype=dtype)
    out = dict(y=z(1, D, T), dx=z(1, C3, T), ds=z(1, C3, T), dk=z(D, Lk), dib=z(C3), dsw=z(C3, 3), dsb=z(C3), dfb=z(D),
               c=[])
    for bk in plan:
        L = bk.L
        kk = _kpad(k, L)
        cb, dkb = z(len(bk.seqs), D, L), z(D, L)
        by_n = {}
        for j, i in enumerate(bk.seqs):
            by_n.setdefault(seqs[i][1], []).append(j)
        for n, js in by_n.items():
            offs = [seqs[bk.seqs[j]][0] for j in js]
            xs = torch.stack([p[0, :, a:a + n] for a in offs])
            ds_ = torch.stack([dy[0, :, a:a + n] for a in offs])
            r = core_ref(xs, ib, sw, sb, kk[:, :n], fb, ds_, dtype=dtype, conv=conv)
            for m, (j, a) in enumerate(zip(js, offs)):
                out["y"][0, :, a:a + n] = r["y"][m]
                out["dx"][0, :, a:a + n] = r["dx"][m]
                out["ds"][0, :, a:a + n] = r["ds"][m]
                cb[j, :, L - n:] = r["c"][m]
            dkb[:, :n] += r["dk"]
            for name in ("dib", "dsw", "dsb", "dfb"):
                out[name] += r[name]
        m = min(L, Lk)
        out["dk"][:, :m] += dkb[:, :m]
        out["c"].append(cb)
    return out


def packed_core_refs(*args, **kw):
    """(fp32 reference, fp64 truth) of packed_core_ref on the host."""
    return packed_core_ref(*args, dtype=torch.float32, **kw), packed_core_ref(*args, dtype=torch.float64, **kw)


def gather_rows(x, seqs, bk):
    """The rows a packed launch sees: row b's position t is x[..., seg_base[b] + t] (0 before the buffer and past it)."""
    C, T = x.shape[1], x.shape[2]
    out = torch.zeros(len(bk.seqs), C, bk.L, dtype=x.dtype)
    for b, sg in enumerate(bk.seg_base):
        lo, hi = max(0, sg), min(T, sg + bk.L)
        out[b, :, lo - sg:hi - sg] = x[0, :, lo:hi]
    return out


def masked_packed(p, ib, sw, sb, k, fb, dy, seqs, plan, bug=None):
    """masked_core on each bucket's rows as the launch sees them (gather_rows: the pads hold the previous sequences'
    samples), outputs scattered back to the real positions: y, dx, c, dk and the parameter gradients of
    packed_core_ref.  bug "start-1": every window reads one position before row_start, the previous sequence's last
    sample."""
    C3, T = p.shape[1], p.shape[2]
    D, Lk = C3 // 3, k.shape[1]
    z = lambda *s: torch.zeros(*s, dtype=torch.float64)
    out = dict(y=z(1, D, T), dx=z(1, C3, T), dk=z(D, Lk), dib=z(C3), dsw=z(C3, 3), dsb=z(C3), dfb=z(D), c=[])
    for bk in plan:
        L = bk.L
        kk = _kpad(k, L)[:, :L]
        r = masked_core(gather_rows(p, seqs, bk), ib, sw, sb, kk, fb, gather_rows(dy, seqs, bk), bk.row_start, bug=bug)
        for b, (i, rs) in enumerate(zip(bk.seqs, bk.row_start)):
            a, n = seqs[i]
            out["y"][0, :, a:a + n] = r["y"][b, :, rs:]
            out["dx"][0, :, a:a + n] = r["dx"][b, :, rs:]
        out["c"].append(r["c"])
        m = min(L, Lk)
        out["dk"][:, :m] += r["dk"][:, :m]
        for name in ("dib", "dsw", "dsb", "dfb"):
            out[name] += r[name]
    return out


def plant(r, bug, seqs, plan, t):
    """A copy of the fp64 packed reference r with one packed-addressing bug planted (the write-side and host-side
    ones; the window read before row_start is masked_packed's "start-1"):
      "ds at start-1" / "dp at start-1": each bucket, in launch order, also writes position row_start - 1 of its rows,
        the last position of the previous sequence: ds there is 0 (dc and dg are masked), dp the unmasked transposed
        filter w1 ds[rs] + w0 ds[rs + 1];
      "seg_base+1": every row addressed one position late (reads and writes shifted, nothing before or after it);
      "dk uncut": a bucket's dk added over its L_b taps, not cut to Lk;
      "dib neighbour": d in_proj.bias also sums the previous sequence's last dp;
      "ds carry": the transposed short filter applied to the whole pack, so the next sequence's first ds reach a
        sequence's last two dp (and d in_proj.bias)."""
    o = {k: ([c.clone() for c in v] if isinstance(v, list) else v.clone()) for k, v in r.items()}
    w = t["sw"].double()
    if bug in ("ds at start-1", "dp at start-1"):
        name = "ds" if bug == "ds at start-1" else "dx"
        o[name].zero_()
        ds = torch.cat([r["ds"][0], torch.zeros(r["ds"].shape[1], 1, dtype=r["ds"].dtype)], 1)
        for bk in plan:                     # launch order: a later launch overwrites an earlier stray write
            for i in bk.seqs:
                a, n = seqs[i]
                o[name][0, :, a:a + n] = r[name][0, :, a:a + n]
            for i in bk.seqs:
                a, n = seqs[i]
                if a > 0:
                    nxt = ds[:, a + 1] if n > 1 else 0.0 * ds[:, a]
                    o[name][0, :, a - 1] = 0.0 if name == "ds" else w[:, 1] * ds[:, a] + w[:, 0] * nxt
    elif bug == "seg_base+1":
        shift = [(a + 1, n) for a, n in seqs]
        pad = lambda x: torch.cat([x, torch.zeros(*x.shape[:-1], 1, dtype=x.dtype)], -1)
        s = packed_core_ref(pad(t["p"]), t["ib"], t["sw"], t["sb"], t["k"], t["fb"], pad(t["dy"]), shift,
                            make_plan(shift, [(bk.L, bk.seqs) for bk in plan]))
        o = dict(s, y=s["y"][..., :-1], dx=s["dx"][..., :-1], ds=s["ds"][..., :-1])
    elif bug == "dk uncut":
        Lmax = max(bk.L for bk in plan)
        o["dk"] = torch.cat([r["dk"], torch.zeros(r["dk"].shape[0], max(0, Lmax - r["dk"].shape[1]), dtype=r["dk"].dtype)], 1)
    elif bug == "dib neighbour":
        for a, n in seqs:
            if a > 0 and n > 0:
                o["dib"] += r["dx"][0, :, a - 1]
    elif bug == "ds carry":
        ds = torch.cat([r["ds"][0], torch.zeros(r["ds"].shape[1], 2, dtype=r["ds"].dtype)], 1)
        full = w[:, 2:3] * ds[:, :-2] + w[:, 1:2] * ds[:, 1:-1] + w[:, 0:1] * ds[:, 2:]
        real = _real_mask(seqs, r["ds"].shape[-1])
        o["dx"] = torch.where(real, full, 0.0)[None]
        o["dib"] = o["dx"][0].sum(1)
    else:
        raise ValueError(bug)
    return o


def _real_mask(seqs, T):
    m = torch.zeros(T, dtype=torch.bool)
    for a, n in seqs:
        m[a:a + n] = True
    return m


def bucket_index(seqs, bk):
    return torch.cat([torch.arange(seqs[i][0], seqs[i][0] + seqs[i][1]) for i in bk.seqs])


def check_packed(o, r32, r64, seqs, plan, tag, names=("y", "c", "ds", "dp"), grads=("dk", "dsw", "dsb", "dfb", "dib")):
    """Every activation per bucket (the real positions of its sequences; c in its row layout), every gradient whole."""
    for k, bk in enumerate(plan):
        idx = bucket_index(seqs, bk)
        bt = f"{tag} L_b={bk.L} rows={len(bk.seqs)}"
        for n in names:
            if n == "c":
                _act(o["c"][k], r32["c"][k], r64["c"][k], f"{bt} c")
            else:
                rn = "dx" if n == "dp" else n
                _act(o[n][..., idx], r32[rn][..., idx], r64[rn][..., idx], f"{bt} {n}")
    for n in grads:
        _par(o[n], r32[n], r64[n], f"{tag} grad {n}")


# ------------------------------------------------------------------------------------------ inputs
def pack_inputs(seqs, T, D, Lk, seed, big=(), gap_fill=None):
    """Seeded host inputs of one packed call: p (1, 3D, T), dy (1, D, T), the core's parameters and a decaying filter k
    (D, Lk).  Sequences in ``big`` hold values of magnitude 3 to 10 (the neighbours a missing predicate would read);
    positions outside every sequence hold ``gap_fill`` (a NaN encoding of tests/test_gpu_widths.NANS, "inf", or a
    number)."""
    g = torch.Generator().manual_seed(seed)
    C3 = 3 * D
    t = dict(p=torch.randn(1, C3, T, generator=g), dy=torch.randn(1, D, T, generator=g),
             ib=torch.randn(C3, generator=g) * 0.5, sw=(torch.rand(C3, 3, generator=g) * 2 - 1) / math.sqrt(3),
             sb=(torch.rand(C3, generator=g) * 2 - 1) / math.sqrt(3), k=decaying_filter(D, Lk, g),
             fb=torch.randn(D, generator=g))
    for i in big:
        a, n = seqs[i]
        for name in ("p", "dy"):
            x = t[name][..., a:a + n]
            t[name][..., a:a + n] = (3 + 7 * torch.rand(x.shape, generator=g)) * torch.randn(x.shape, generator=g).sign()
    if gap_fill is not None:
        gap = ~_real_mask(seqs, T)
        for name in ("p", "dy"):
            v = (_poison(t[name], gap_fill, g) if isinstance(gap_fill, str)
                 else torch.full_like(t[name], float(gap_fill)))
            t[name] = torch.where(gap, v, t[name])
    return t


ARGS = ("p", "ib", "sw", "sb", "k", "fb", "dy")


# ------------------------------------------------------------------------------------------ sweep and test layouts
SWEEP_LB = [1 << e for e in range(10, 21)]
SINGLE_ROW_LB = SWEEP_LB
# odd L at every LOGM1 through the C ABI, L % 4 == 2, and L < 1024 (LOGM1 = 0)
ABI_L = [1, 2, 3, 5, 255, 1022, 1023, 2047, 4095, 8191, 16383, 32767, 40002, 65535, 131071, 262143, 524287, 1048575]


def sweep_pack(L, i):
    """Sequences of bucket L_b = L with row_start = L - n on every packed_starts(L), interleaved with short neighbours
    of another bucket (1024, or 2048 when L = 1024) holding large values; the first sequence sits at offset 0 with a
    negative seg_base, the last ends at total, and total % 4 == i % 4.  -> (seqs, target indices, neighbour indices,
    neighbour bucket)."""
    starts = packed_starts(L)
    starts = starts[1:] + starts[:1]                # a start > 0 first: seg_base = -row_start < 0 at offset 0
    nbL = 2048 if L == 1024 else 1024
    nb_n = [1025, 2047, 1500, 2048] if nbL == 2048 else [1, 2, 3, 517, 1023, 700]
    lengths, tg, nb = [], [], []
    for j, s in enumerate(starts):
        tg.append(len(lengths)); lengths.append(L - s)
        nb.append(len(lengths)); lengths.append(nb_n[j % len(nb_n)])
    lengths[-1] = nb_n[-1]
    lengths[-1] -= (sum(lengths) - i) % 4
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    return seqs_from_cu(cu), tg, nb, nbL


def decisions_sweep(L, i):
    """Cells of the coverage table the sweep pack at L reaches."""
    g = packed_geometry(L)
    seqs, tg, _, _ = sweep_pack(L, i)
    starts = {L - seqs[j][1] for j in tg}
    b, m = g["boundaries"], g["logm1"]
    out = {("fwd", m, "L%4==0"), ("bwd", m, "L%4==0"), ("total % 4", sum(n for _, n in seqs) % 4)}
    if g["two"] and all(b["tile"][0] + d in starts for d in range(-2, 3)):
        out.add(("tile halo", m))
    if any(r in starts for r in b["row"]):
        out.add(("column-row edge", m))
    if b["pair_bwd"] and all(b["pair_bwd"][0] + d in starts for d in range(-2, 3)):
        out.add(("two-slot batch edge", m))
    if b["span"] and b["span"][0] in starts and b["span"][-1] in starts:
        out.add(("span first and last", m))
    return out


def decisions_abi(L):
    g = masked_geometry(L)
    kind = "L%4==0" if L % 4 == 0 else ("odd" if L % 2 else "L%4==2")
    out = {("fwd", g["logm1"], kind), ("bwd", g["logm1"], kind), ("c_save", "vec" if L % 2 == 0 else "scalar")}
    if L < 1024:
        out.add(("L < 1024",))
    return out


# ------------------------------------------------------------------------------------------ CPU self-checks
def test_coverage_table():
    """The packed sweep and the C ABI cases reach every LOGM1 in both directions with L % 4 == 0 (host-planned bucket
    lengths) and odd L, and on every TWO size row starts on the first tile edge's halo and the first two-slot batch
    edge; column-row edges and the first and last short_conv_bwd span wherever the bucket has them; every residue of
    total mod 4; B = 1 with and without a saved spectrum at every LOGM1."""
    hit = set()
    for i, L in enumerate(SWEEP_LB):
        hit |= decisions_sweep(L, i)
    for L in ABI_L:
        hit |= decisions_abi(L)
    for L in SINGLE_ROW_LB:
        hit |= {("B=1", masked_geometry(L)["logm1"], s) for s in ("saved", "recompute")}
    want = {(d, m, kind) for d in ("fwd", "bwd") for m in range(11) for kind in ("L%4==0", "odd")}
    want |= {(cell, m) for cell in ("tile halo", "two-slot batch edge") for m in range(5, 11)}
    want |= {("column-row edge", m) for m in range(2, 11)} | {("span first and last", m) for m in range(4, 11)}
    want |= {("total % 4", r) for r in range(4)} | {("c_save", "vec"), ("c_save", "scalar"), ("L < 1024",)}
    want |= {("B=1", m, s) for m in range(11) for s in ("saved", "recompute")}
    assert not want - hit, f"table cells not hit: {sorted(want - hit, key=str)}"
    # the geometry the cells rest on: two slots per packed backward batch, so its first edge at 2^20 is 2048 * 2 * 32
    assert packed_epilogue_slots() == 2
    assert packed_geometry(1 << 20)["boundaries"]["pair_bwd"][0] == 131072
    assert packed_geometry(1 << 15)["boundaries"]["pair_bwd"][:2] == [4096, 8192]
    for i, L in enumerate(SWEEP_LB):            # the sweep pack's layout promises
        seqs, tg, nb, nbL = sweep_pack(L, i)
        assert seqs[0][0] == 0 and L - seqs[0][1] > 0 and all(ops.bucket_length(seqs[j][1]) == nbL for j in nb)
        assert sorted(L - seqs[j][1] for j in tg) == packed_starts(L)
    for L in ABI_L:
        assert abi_starts(L) and all(0 <= s < L for s in abi_starts(L))


def _small_pack(D=3, seed=5):
    """Two hand-made buckets (L_b = 32 and 48) interleaved, neighbours large, a longer sequence after a shorter one (so
    a stray write at row_start - 1 lands in a bucket that launched earlier)."""
    cu = [0]
    for n in [5, 40, 1, 33, 2, 47, 17, 3]:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = make_plan(seqs, [(32, [i for i, (_, n) in enumerate(seqs) if n <= 32]),
                            (48, [i for i, (_, n) in enumerate(seqs) if n > 32])])
    return seqs, plan, pack_inputs(seqs, cu[-1], D, 47, seed, big=(0, 2, 4))


def test_packed_ref_is_rows_ref_and_masked_core():
    """packed_core_ref against rows_core_ref on each bucket's left-padded rows (the pads zero, then holding the previous
    sequences' samples as a launch sees them) and against masked_core on those rows; O(n^2) time-domain and
    O.fftconv_ref convolutions give the same."""
    seqs, plan, t = _small_pack()
    args = [t[n] for n in ARGS]
    r = packed_core_ref(*args, seqs, plan)
    for k, bk in enumerate(plan):
        rows = rows_core_ref(gather_rows(t["p"], seqs, bk), *args[1:4], _kpad(t["k"], bk.L)[:, :bk.L], t["fb"],
                             gather_rows(t["dy"], seqs, bk), bk.row_start)
        for b, (i, rs) in enumerate(zip(bk.seqs, bk.row_start)):
            a, n = seqs[i]
            for name in ("y", "dx", "ds"):
                torch.testing.assert_close(rows[name][b, :, rs:], r[name][0, :, a:a + n], rtol=1e-10, atol=1e-10)
        torch.testing.assert_close(rows["c"], r["c"][k], rtol=1e-10, atol=1e-10)
    m = masked_packed(*args, seqs, plan)
    for name in ("y", "dx", "dk", "dib", "dsw", "dsb", "dfb"):
        torch.testing.assert_close(m[name], r[name], rtol=1e-10, atol=1e-10, msg=name)
    for k in range(len(plan)):
        torch.testing.assert_close(m["c"][k], r["c"][k], rtol=1e-10, atol=1e-10)
    for conv in (O.fftconv_direct, O.fftconv_ref):
        d = packed_core_ref(*args, seqs, plan, conv=conv)
        for name in ("y", "dx", "ds", "dk", "dib", "dsw", "dsb", "dfb"):
            torch.testing.assert_close(d[name], r[name], rtol=1e-10, atol=1e-10, msg=f"{conv.__name__} {name}")


PLANTED = ["read before start", "ds at start-1", "dp at start-1", "seg_base+1", "dk uncut", "dib neighbour", "ds carry"]


@pytest.mark.parametrize("bug", PLANTED)
def test_parity_bar_rejects_planted_packed_bugs(bug):
    """Each planted packing bug is rejected by the bar that the unplanted packed reference passes.  The filter has
    Lk = 47 taps, shorter than the 48-sample bucket, so a dk not cut to Lk shows."""
    seqs, plan, t = _small_pack()
    args = [t[n] for n in ARGS]
    r32, r64 = packed_core_refs(*args, seqs, plan)
    n0 = len(PU._records)

    def bar(o):
        check_packed(dict(o, dp=o["dx"]), r32, r64, seqs, plan, f"planted {bug}",
                     names=("y", "c", "ds", "dp") if "ds" in o else ("y", "c", "dp"))

    try:
        bar(r64)
        bar(masked_packed(*args, seqs, plan))
        with pytest.raises(AssertionError):
            if bug == "read before start":
                bar(masked_packed(*args, seqs, plan, bug="start-1"))
            else:
                bar(plant(r64, bug, seqs, plan, t))
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


def _sentinel(shape, dev):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def packed_run(H, t, plan, dev, c_off=0, on_device=False):
    """The three packed entry points per bucket, in plan order, as ops.core_forward_packed / core_backward_packed call
    them (ops.workspace, ops._save_spectrum, ops._bucket_filter, dk summed over min(L_b, Lk)), with caller-owned y_pre,
    c, ds and dp pre-filled with SENTINEL; c at c_off bytes past an aligned allocation.  Returns every output (on the
    host unless on_device)."""
    lib, P = H._lib.lib(), ops._ptr
    p, ib, sw, sb, k, fb, dy = (t[n] if on_device else t[n].to(dev) for n in ARGS)
    sg, rs = ops._bucket_tables(plan, dev)
    _, C3, T = p.shape
    D, Lk = C3 // 3, k.shape[1]
    y, ds, dp = _sentinel((1, D, T), dev), _sentinel((1, C3, T), dev), _sentinel((1, C3, T), dev)
    dk = torch.zeros(D, Lk, device=dev)
    dsw, dsb, dfb, dib = (torch.zeros(*s, device=dev) for s in ((C3, 3), (C3,), (D,), (C3,)))
    saved = []
    for bk in plan:
        B, L = len(bk.seqs), bk.L
        kspec = ops.filter_spectrum(ops._bucket_filter(k, L))
        c = _sentinel((B, D, L), dev)
        if c_off:
            c = _at_offset(c, c_off)
        gs = torch.empty(D * B, kspec.shape[-1], dtype=torch.complex64, device=dev) if ops._save_spectrum() else None
        ws = ops.workspace(B, D, L, False, dev)
        H._lib.check(lib.hyena_b200_core_fwd_packed(P(p), P(ib), P(sw), P(sb), P(kspec), P(fb), P(y), P(c), P(gs),
                                                    P(sg[bk.offset:]), P(rs[bk.offset:]), T, B, D, L, P(ws), ws.numel(),
                                                    ops._stream()))
        saved.append((kspec, c, gs))
    for bk, (kspec, c, gs) in zip(plan, saved):
        B, L = len(bk.seqs), bk.L
        dkb = torch.empty(D, L, device=dev)
        ws = ops.workspace(B, D, L, True, dev)
        H._lib.check(lib.hyena_b200_core_bwd_packed(P(dy), P(p), P(ib), P(sw), P(sb), P(kspec), P(fb), P(c), P(gs),
                                                    P(dkb), P(dsw), P(dsb), P(dfb), P(ds), P(sg[bk.offset:]),
                                                    P(rs[bk.offset:]), T, B, D, L, P(ws), ws.numel(), ops._stream()))
        H._lib.check(lib.hyena_b200_short_bwd_packed(P(ds), P(sw), P(dp), P(dib), P(sg[bk.offset:]), P(rs[bk.offset:]),
                                                     T, B, C3, L, ops._stream()))
        m = min(L, Lk)
        dk[:, :m] += dkb[:, :m]
    torch.cuda.synchronize()
    o = dict(y=y, ds=ds, dp=dp, dk=dk, dsw=dsw, dsb=dsb, dfb=dfb, dib=dib, c=[s[1] for s in saved])
    if on_device:
        return o
    return {n: ([x.cpu() for x in v] if isinstance(v, list) else v.cpu()) for n, v in o.items()}


def ops_run(H, t, plan, dev):
    """ops.core_forward_packed / core_backward_packed on the same plan: y, c, dp, dk and the sums on the host."""
    p, ib, sw, sb, k, fb, dy = (t[n].to(dev) for n in ARGS)
    tables = ops._bucket_tables(plan, dev)
    y, saved = ops.core_forward_packed(p, ib, sw, sb, k, fb, plan, tables, True)
    dp, dk, dsw, dsb, dfb, dib = ops.core_backward_packed(dy, p, ib, sw, sb, fb, k.shape[1], plan, tables, saved)
    torch.cuda.synchronize()
    return dict(y=y.cpu(), c=[s[1].cpu() for s in saved], dp=dp.cpu(), dk=dk.cpu(), dsw=dsw.cpu(), dsb=dsb.cpu(),
                dfb=dfb.cpu(), dib=dib.cpu())


def _bits(x):
    return x.contiguous().view(torch.int32)


def check_untouched(o, seqs, plan, tag):
    """Positions outside every sequence keep the sentinel's bits in y_pre, ds and dp; c is exactly 0 at t < row_start."""
    gap = ~_real_mask(seqs, o["y"].shape[-1])
    for n in ("y", "ds", "dp"):
        assert bool((_bits(o[n])[..., gap] == SENTINEL).all()), f"{tag}: {n} written outside the sequences"
    for k, bk in enumerate(plan):
        for b, rs in enumerate(bk.row_start):
            assert not bool(o["c"][k][b, :, :rs].any()), f"{tag}: c of L_b={bk.L} row {b} is not 0 before row_start {rs}"


def run_and_check(H, dev, t, seqs, plan, tag, refs=None, **kw):
    r32, r64 = refs or packed_core_refs(*(t[n] for n in ARGS), seqs, plan)
    o = packed_run(H, t, plan, dev, **kw)
    check_packed(o, r32, r64, seqs, plan, tag)
    check_untouched(o, seqs, plan, tag)
    return o, (r32, r64)


# ------------------------------------------------------------------------------------------ 1. transform size sweep
@gpu
@pytest.mark.parametrize("L", SWEEP_LB)
def test_packed_core_sweep(L):
    """Bucket L_b = L with its sequences' row starts on every packed_starts(L), interleaved with short neighbours of
    another bucket, D = 2.  The two buckets launch in increasing (the host plan's) and in decreasing order, both against
    the per-sequence truth; the increasing order also gives ops.core_forward_packed / core_backward_packed's bits."""
    H = _H()
    dev = _dev()
    i = SWEEP_LB.index(L)
    seqs, tg, nb, nbL = sweep_pack(L, i)
    T = seqs[-1][0] + seqs[-1][1]
    t = pack_inputs(seqs, T, 2, max(n for _, n in seqs), seed=101 * i, big=nb)
    up = make_plan(seqs, sorted([(L, tg), (nbL, nb)]))
    o, refs = run_and_check(H, dev, t, seqs, up, f"packed sweep L_b={L} increasing")
    down = make_plan(seqs, sorted([(L, tg), (nbL, nb)], reverse=True))
    run_and_check(H, dev, t, seqs, down, f"packed sweep L_b={L} decreasing", refs=(
        {**refs[0], "c": refs[0]["c"][::-1]}, {**refs[1], "c": refs[1]["c"][::-1]}))
    via = ops_run(H, t, up, dev)
    for n in ("y", "dp", "dk"):
        assert torch.equal(via[n], o[n]), f"L_b={L}: ops route {n} differs"
    for k in range(len(up)):
        assert torch.equal(via["c"][k], o["c"][k]), f"L_b={L}: ops route c differs"


# ------------------------------------------------------------------------------------------ 2. single-row buckets
@gpu
@pytest.mark.parametrize("L", SINGLE_ROW_LB)
def test_packed_single_row(monkeypatch, L):
    """One sequence in bucket L (row start L/4 + 1) between short neighbours: with the g spectrum saved (ROW_CONV_BWD1
    for the single row) and with HYENA_B200_SAVE_SPECTRUM=0 (COL_GATE_PACKED again in the backward, ROW_CONV_BWD)."""
    H = _H()
    dev = _dev()
    nbL = 2048 if L == 1024 else 1024
    lengths = [1025, L - L // 4 - 1, 1500] if nbL == 2048 else [3, L - L // 4 - 1, 700, 1]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = make_plan(seqs, sorted([(L, [1]), (nbL, [j for j in range(len(seqs)) if j != 1])]))
    t = pack_inputs(seqs, cu[-1], 2, max(lengths), seed=7 * L, big=[j for j in range(len(seqs)) if j != 1])
    refs = None
    for save in ("1", "0"):
        monkeypatch.setenv("HYENA_B200_SAVE_SPECTRUM", save)
        H._lib.profile_begin()
        _, refs = run_and_check(H, dev, t, seqs, plan, f"packed B=1 L_b={L} spectrum={save}", refs=refs)
        prof = H._lib.profile_end()
        assert prof["col_fwd<gate>"][1] == (2 if save == "1" else 4), prof


# ------------------------------------------------------------------------------------------ 3. channel groups
@gpu
def test_packed_channel_groups(monkeypatch):
    """The workspace cut to 3 channels per launch (D = 7: 3 + 3 + 1, c0 > 0, a ragged last group) on two buckets: every
    output against the truth, and bit for bit the one-group run (the atomic sums against the truth only)."""
    H = _H()
    dev = _dev()
    cu = [0]
    for n in [5, 3000, 1, 1024, 2049, 77, 4096]:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = ops.packed_plan(cu)
    t = pack_inputs(seqs, cu[-1], 7, 4096, seed=59)
    base, refs = run_and_check(H, dev, t, seqs, plan, "packed groups one group")
    monkeypatch.setattr(ops, "workspace", _exact_workspace(H, 3))
    H._lib.profile_begin()
    got, _ = run_and_check(H, dev, t, seqs, plan, "packed groups G=3", refs=refs)
    prof = H._lib.profile_end()
    n = {k: v[1] for k, v in prof.items()}
    assert n["col_fwd<gate>"] == 6 and n["col_fwd<dc>"] == 6 and n["col_inv<bwd_dg>"] == 6, n
    assert n["short_conv_bwd"] == 2, n
    for name in ("y", "ds", "dp", "dk"):
        assert torch.equal(got[name], base[name]), f"packed groups: {name} differs from the one-group run"
    for k in range(len(plan)):
        assert torch.equal(got["c"][k], base["c"][k]), "packed groups: c differs from the one-group run"


@gpu
def test_packed_natural_group_cut():
    """4,096 sequences of one bucket at D = 16: 65535 // 4096 = 15 channels per launch, so the bucket runs as 15 + 1.
    Every output against the truth; the first 100 sequences' y_pre, ds and dp bit for bit those of a pack of them
    alone, which runs as one group."""
    H = _H()
    dev = _dev()
    D = 16
    lengths = [1 + (37 * i) % 61 for i in range(4096)]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = ops.packed_plan(cu)
    assert len(plan) == 1
    t = pack_inputs(seqs, cu[-1], D, 61, seed=61)
    H._lib.profile_begin()
    o, _ = run_and_check(H, dev, t, seqs, plan, "packed natural groups")
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 2 and prof["col_inv<dk>"][1] == 2, prof
    m = cu[100]
    sub = dict(t, p=t["p"][..., :m].contiguous(), dy=t["dy"][..., :m].contiguous())
    H._lib.profile_begin()
    s = packed_run(H, sub, ops.packed_plan(cu[:101]), dev)
    assert H._lib.profile_end()["col_fwd<gate>"][1] == 1
    for name in ("y", "ds", "dp"):
        assert torch.equal(s[name], o[name][..., :m]), f"natural groups: {name} of the first 100 sequences differs"


# ------------------------------------------------------------------------------------------ 4. split bucket
@gpu
def test_packed_split_bucket():
    """65,535 + 5 sequences of lengths 1 to 3 at D = 2: ops.packed_plan splits the bucket, the first part runs one
    channel per launch (65535 // 65535), the second reads its tables at bk.offset = 65535.  Against the truth (batched by
    length), through the entry points and through ops."""
    H = _H()
    dev = _dev()
    N = ops.MAX_BUCKET_ROWS + 5
    lengths = [1 + (i * 7) % 3 for i in range(N)]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = ops.packed_plan(cu)
    assert [len(b.seqs) for b in plan] == [ops.MAX_BUCKET_ROWS, 5] and plan[1].offset == ops.MAX_BUCKET_ROWS
    t = pack_inputs(seqs, cu[-1], 2, 3, seed=67)
    H._lib.profile_begin()
    o, refs = run_and_check(H, dev, t, seqs, plan, "packed split bucket")
    prof = H._lib.profile_end()
    assert prof["col_fwd<gate>"][1] == 3 and prof["short_conv_bwd"][1] == 2, prof
    via = ops_run(H, t, plan, dev)
    for n in ("y", "dp", "dk"):
        assert torch.equal(via[n], o[n]), f"split bucket: ops route {n} differs"
    for n in ("dsw", "dsb", "dfb", "dib"):
        _par(via[n], refs[0][n], refs[1][n], f"packed split bucket ops grad {n}")


# ------------------------------------------------------------------------------------------ 5. 64-bit offsets
@gpu
def test_packed_64bit_offsets():
    """D = 256, sequences of 2^20 - 1, 2^20, 2^20 - 3 and 1,000 positions: total = 3,146,724, so the v rows 2D + c of
    every channel c >= 171 lie wholly past element 2^31.  y_pre, c, ds, dp and the per-channel gradients of channels 0,
    170, 171, 200 and 255 (the last channel group of the 2^20 bucket) against the truth of those channels alone (the
    core is depthwise)."""
    H = _H()
    dev = _dev()
    D = 256
    lengths = [(1 << 20) - 1, 1 << 20, (1 << 20) - 3, 1000]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    T = cu[-1]
    seqs = seqs_from_cu(cu)
    assert (2 * D + 170) * T < 2 ** 31 <= (2 * D + 171) * T
    plan = ops.packed_plan(cu)
    g = torch.Generator(device=dev).manual_seed(71)
    gh = torch.Generator().manual_seed(72)
    t = dict(p=torch.randn(1, 3 * D, T, generator=g, device=dev), dy=torch.randn(1, D, T, generator=g, device=dev),
             ib=(torch.randn(3 * D, generator=gh) * 0.5).to(dev),
             sw=((torch.rand(3 * D, 3, generator=gh) * 2 - 1) / math.sqrt(3)).to(dev),
             sb=((torch.rand(3 * D, generator=gh) * 2 - 1) / math.sqrt(3)).to(dev),
             k=decaying_filter(D, 1 << 20, gh).to(dev), fb=torch.randn(D, generator=gh).to(dev))
    try:
        o = packed_run(H, t, plan, dev, on_device=True)
        chans = [0, 170, 171, 200, 255]
        rows = [c + j * D for j in range(3) for c in chans]
        sub = dict(p=t["p"][:, rows].cpu(), dy=t["dy"][:, chans].cpu(), ib=t["ib"][rows].cpu(),
                   sw=t["sw"][rows].cpu(), sb=t["sb"][rows].cpu(), k=t["k"][chans].cpu(), fb=t["fb"][chans].cpu())
        got = dict(y=o["y"][:, chans].cpu(), ds=o["ds"][:, rows].cpu(), dp=o["dp"][:, rows].cpu(),
                   c=[c[:, chans].cpu() for c in o["c"]], dk=o["dk"][chans].cpu(), dsw=o["dsw"][rows].cpu(),
                   dsb=o["dsb"][rows].cpu(), dfb=o["dfb"][chans].cpu(), dib=o["dib"][rows].cpu())
    finally:
        t = o = None
        ops._ws_cache.clear()
        torch.cuda.empty_cache()
    r32, r64 = packed_core_refs(*(sub[n] for n in ARGS), seqs, plan)
    check_packed(got, r32, r64, seqs, plan, "packed 64-bit channels 0/170/171/200/255")


# ------------------------------------------------------------------------------------------ 6. the C ABI contract
def abi_layout(L, starts, seed):
    """One bucket of rows of length L with the given row starts: sequences of n = L - s positions laid out with gaps of
    1 to 4 positions between them (and before the first and after the last), rows listed in an order that is not
    their order in the buffer.  -> (seqs, plan, T)."""
    g = torch.Generator().manual_seed(seed)
    seqs, a = [], 0
    for s in starts:
        a += 1 + int(torch.randint(0, 4, (1,), generator=g))
        seqs.append((a, L - s)); a += L - s
    T = a + 1 + int(torch.randint(0, 4, (1,), generator=g))
    order = torch.randperm(len(seqs), generator=g).tolist()
    return seqs, make_plan(seqs, [(L, order)]), T


@gpu
@pytest.mark.parametrize("L", ABI_L)
def test_abi_lengths(L):
    """Any L through the C entry points, with hand-made seg_base / row_start tables (abi_starts) over gaps that hold
    NaN or +-inf in p and dy_pre: every position outside the sequences keeps the sentinel's bits in y_pre, ds and dp, c
    is exactly 0 before each row start, everything inside is finite and within the bar, and the atomically reduced sums
    are held to the fp64 truth."""
    H = _H()
    dev = _dev()
    starts = abi_starts(L)
    seqs, plan, T = abi_layout(L, starts, seed=L)
    fill = [*NANS, "inf"][L % 4]
    t = pack_inputs(seqs, T, 2, L, seed=3 * L + 1, big=range(0, len(seqs), 2), gap_fill=fill)
    run_and_check(H, dev, t, seqs, plan, f"abi L={L} gaps {fill}")


@gpu
@pytest.mark.parametrize("L", [1024, 40000])
def test_abi_c_save_offset(L):
    """c_save 4 bytes off an 8-byte boundary: vec = 0 (scalar c accesses) at an even L."""
    H = _H()
    dev = _dev()
    seqs, plan, T = abi_layout(L, abi_starts(L), seed=L + 5)
    t = pack_inputs(seqs, T, 2, L, seed=L + 6, big=range(1, len(seqs), 2), gap_fill="inf")
    run_and_check(H, dev, t, seqs, plan, f"abi L={L} c at +4 bytes", c_off=4)


# ------------------------------------------------------------------------------------------ 7. neighbour contents
@gpu
@pytest.mark.parametrize("L", [1 << 15, 1 << 20])
def test_packed_neighbour_contents(L):
    """A sequence of bucket L (row start 3) between neighbours of bucket 1024 whose p and dy_pre hold zeros, random
    values, the NaN encodings and +-inf: the target's y_pre, c and ds keep their bits (the host plan, one launch per
    pass per bucket); with zero neighbours, everything against the truth."""
    H = _H()
    dev = _dev()
    cu = [0]
    for n in [5, L - 3, 700, 2]:
        cu.append(cu[-1] + n)
    seqs = seqs_from_cu(cu)
    plan = ops.packed_plan(cu)
    t0 = pack_inputs(seqs, cu[-1], 2, L - 3, seed=79)
    nbr = ~_real_mask([seqs[1]], cu[-1])

    def filled(fill):
        g = torch.Generator().manual_seed(83 + (fill if isinstance(fill, int) else 0))
        out = dict(t0)
        for name in ("p", "dy"):
            x = t0[name]
            if fill == "zero":
                v = torch.zeros_like(x)
            elif isinstance(fill, int):
                v = (3 + 7 * torch.rand(x.shape, generator=g)) * torch.randn(x.shape, generator=g).sign()
            else:
                v = _poison(x, fill, g)
            out[name] = torch.where(nbr, v, x)
        return out

    zero, _ = run_and_check(H, dev, filled("zero"), seqs, plan, f"neighbours zero L_b={L}")
    a, n = seqs[1]
    k = [b.L for b in plan].index(L)
    for fill in (1, 2, *NANS, "inf"):
        o = packed_run(H, filled(fill), plan, dev)
        for name in ("y", "ds"):
            assert torch.equal(o[name][..., a:a + n], zero[name][..., a:a + n]), f"L_b={L} {fill}: target {name} changed"
        assert torch.equal(o["c"][k], zero["c"][k]), f"L_b={L} {fill}: target c changed"


# ------------------------------------------------------------------------------------------ 8. operator at d_model 1..3
@gpu
@pytest.mark.parametrize("D", [1, 2, 3])
def test_packed_operator_small_widths(D):
    """HyenaOperator(u, cu_seqlens=) at d_model 1, 2 and 3 (no LayerNorm) against the per-sequence fp64 truth at the
    full bar; the left-padded operator (mask=) on the same sequences is held to the same bar."""
    from tests.test_gpu_ragged import _make
    from tests.test_gpu_ragged_train import _mask
    from tests.test_gpu_varlen import _check_truth, _train
    from tests.test_varlen_cpu import packed_input, seq_truth
    dev = _dev()
    n0 = len(PU._records)
    lengths = [700, 1, 1025, 3, 4096, 33, 2048, 2, 4095]
    op, P = _make(D, 4096, seed=D)
    u, cu = packed_input(lengths, D, seed=D)
    dy = torch.randn(u.shape, generator=torch.Generator().manual_seed(90 + D))
    _check_truth(_train(op, u, dy, torch.tensor(cu, dtype=torch.int32)), u, dy, cu, P, f"packed operator D={D}")
    Pm = max(lengths)
    up, dyp = torch.zeros(len(lengths), Pm, D), torch.zeros(len(lengths), Pm, D)
    for b, (a, e) in enumerate(zip(cu[:-1], cu[1:])):
        up[b, Pm - (e - a):] = u[a:e]
        dyp[b, Pm - (e - a):] = dy[a:e]
    op.zero_grad(set_to_none=True)
    ud = up.to(dev).requires_grad_(True)
    y = op(ud, mask=_mask(lengths, Pm).to(dev))
    y.backward(dyp.to(dev))
    t32 = seq_truth(u, dy, cu, P, torch.float32, dev)
    t64 = seq_truth(u, dy, cu, P, torch.float64, dev)
    for b, (a, e) in enumerate(zip(cu[:-1], cu[1:])):
        n = e - a
        PU.check(y[b, Pm - n:], t32[0][b], f"left-padded operator D={D} y seq {b} length {n}", ref64=t64[0][b])
        PU.check(ud.grad[b, Pm - n:], t32[1][b], f"left-padded operator D={D} du seq {b} length {n}", ref64=t64[1][b])
    for route in ("packed", "left-padded"):         # the error of each route against fp64, relative to the fp32 oracle's
        rec = [r for r in PU._records[n0:] if r["what"].startswith(route) and " grad " not in r["what"]]
        print(f"\n{route} operator D={D}: {len(rec)} activation comparisons, largest |ours - fp64| / |fp32 oracle - fp64| "
              f"{max(r['e_ours64'] / max(r['e_ref64'], 1e-30) for r in rec):.2f}, largest normwise "
              f"{max(r['normwise'] for r in rec):.2e}, elements missing the bound vs fp64: ours "
              f"{max(r['frac_ours64'] for r in rec):.1e} / fp32 oracle {max(r['frac_ref64'] for r in rec):.1e}")
