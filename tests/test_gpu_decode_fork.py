"""Branched decode caches (DecodeCache.fork / select, ops.decode_branch_step / decode_branch_extend, csrc/decode.cuh
decode_branch_step_kernel and csrc/decode_extend.cuh decode_branch_combine_kernel) through HyenaOperator / Backbone, against
the fp64 truth of the oracle on prefix || branch suffix.  Tolerance policy: tests/parity_util.py."""
import os
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _make(D, l_max, order=2, seed=0, **kw):
    g = torch.Generator().manual_seed(seed)
    P = O.init_params(D, l_max, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    P["in_proj.bias"] = 0.02 * torch.randn(P["in_proj.bias"].shape, generator=g)
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = _H().HyenaOperator(D, l_max, order=order, emb_dim=5, w=10.0, **kw)
    op.load_state_dict(sd)
    if not kw.get("bias", True):
        P["filter_fn.bias"] = torch.zeros_like(P["filter_fn.bias"])
    return op.to(_dev()), P


def _drive(m, cache, u, sched):
    """Feed u (R, m, D) on the GPU to the branched cache by the schedule [(how, n), ...]: step / extend (the route rule) /
    fft / direct (an extend forced onto that route) -> outputs (R, m, D)."""
    ops = _H().ops
    outs, s = [], 0
    with torch.no_grad():
        for how, n in sched:
            if how == "step":
                outs += [m.step(u[:, i:i + 1], cache) for i in range(s, s + n)]
            elif how in ("fft", "direct"):
                outs.append(m._extend(u[:, s:s + n], cache.for_module(m), partial(ops.decode_branch_extend,
                                                                                   fft=how == "fft")))
            else:
                outs.append(m.extend(u[:, s:s + n], cache))
            s += n
    return torch.cat(outs, dim=1)


def _inputs(B, t0, rows, m, D):
    up = O.nucleotide_activations(B, t0, D)[0]
    ub = O.nucleotide_activations(len(rows), m, D, seed=77)[0]
    return up, ub, torch.cat([up[rows], ub], dim=1)


def _check(y, seq, t0, sched, P, what, normalized=False):
    y32 = O.hyena_operator(seq, P, normalized=normalized)[:, t0:]
    y64 = O.hyena_operator(seq.double(), O.to_dtype(P, torch.float64), normalized=normalized)[:, t0:]
    s = 0
    for how, n in sched:
        PU.check(y[:, s:s + n].cpu(), y32[:, s:s + n], f"{what} {how} [{t0 + s}, {t0 + s + n})", ref64=y64[:, s:s + n])
        s += n


def _forked(op, up, t0, rows, horizon, lcap):
    cache = op.allocate_decode_cache(up.shape[0], lcap)
    with torch.no_grad():
        op.prefill(up[:, :t0].to(_dev()), cache)
    return cache, cache.fork(rows, horizon)


def _sched_to(n_total):
    """A mixed step / extend schedule of exactly n_total positions: both extend routes, n = 1 extends, a run of steps."""
    base = [("step", 2), ("direct", 7), ("step", 1), ("fft", 9), ("extend", 1), ("extend", 8)]
    out, left = [], n_total
    for how, n in base:
        if left <= 0:
            break
        out.append((how, min(n, left)))
        left -= min(n, left)
    if left > 0:
        out.append(("step", min(left, 5)))
        left -= min(left, 5)
    if left > 0:
        out.append(("extend", left))
    return out


@pytest.mark.parametrize("B,K,D,t0,mixed", [(1, 1, 32, 1021, False), (1, 4, 32, 1022, False), (1, 9, 256, 1023, False),
                                            (3, 4, 32, 1024, True), (3, 9, 32, 1025, True), (3, 1, 256, 1026, False),
                                            (1, 4, 32, 3, False), (3, 9, 32, 6, True)])
def test_fork_shapes(B, K, D, t0, mixed):
    """K branches per parent for B parents, rows mixed across parents or grouped, t0 at every residue mod 4 and on both sides of
    the 1024-position chunk boundary (and b = 0), run exactly to base + Hc; one more position raises, state untouched."""
    horizon = 48
    rows = [i % B for i in range(B * K)] if mixed else [p for p in range(B) for _ in range(K)]
    b = t0 - t0 % 4
    m = b + horizon - t0
    op, P = _make(D, t0 + m + 64)
    up, ub, seq = _inputs(B, t0, rows, m, D)
    _, br = _forked(op, up, t0, rows, horizon, t0 + m + 64)
    assert (br.base, br.hc) == (b, horizon)
    sched = _sched_to(m)
    y = _drive(op, br, ub.to(_dev()), sched)
    assert br.t == b + horizon
    _check(y, seq, t0, sched, P, f"fork B{B} K{K} D{D} t0 {t0}")
    h0, tail0 = br.h.clone(), br.tail.clone()
    with torch.no_grad():
        for call in (lambda: op.step(ub[:, :1].to(_dev()), br), lambda: op.extend(ub[:, :2].to(_dev()), br)):
            with pytest.raises(_H().HyenaB200Error, match="horizon"):
                call()
    assert br.t == b + horizon and torch.equal(br.h, h0) and torch.equal(br.tail, tail0)


def test_both_routes_at_the_same_positions():
    """Direct and FFT route at the same (t, n) inside a branch, both against fp64 truth and against each other."""
    D, t0, rows = 64, 2050, [0, 0, 1]
    op, P = _make(D, 3000)
    up, ub, seq = _inputs(2, t0, rows, 600, D)
    ys = []
    for route in ("direct", "fft"):
        _, br = _forked(op, up, t0, rows, 1024, 3000)
        sched = [("step", 3), (route, 30), ("step", 1), (route, 566)]
        ys.append(_drive(op, br, ub.to(_dev()), sched))
        _check(ys[-1], seq, t0, sched, P, f"route {route}")
    PU.check(ys[1].cpu(), ys[0].cpu(), "FFT against direct route on a branch")


@pytest.mark.parametrize("variant", ["order3", "order4", "normalized", "trainable_deltas", "no_bias"])
def test_fork_filter_variants(variant):
    D, t0, rows, m = 32, 301, [0, 1, 1], 40
    kw, order, normalized = {}, 2, False
    if variant in ("order3", "order4"):
        order = int(variant[-1])
    elif variant == "normalized":
        kw, normalized = {"normalized": True}, True
    elif variant == "trainable_deltas":
        kw = {"modulation_lr": 1e-3}
    elif variant == "no_bias":
        kw = {"bias": False}
    op, P = _make(D, 400, order=order, **kw)
    up, ub, seq = _inputs(2, t0, rows, m, D)
    _, br = _forked(op, up, t0, rows, 64, 400)
    sched = [("step", 3), ("direct", 12), ("fft", 5), ("step", 2), ("extend", 18)]
    y = _drive(op, br, ub.to(_dev()), sched)
    assert tuple(br.f.shape) == (order - 1, 2, D, 64)
    _check(y, seq, t0, sched, P, f"fork {variant}", normalized)


def test_snapshot_semantics():
    """After the fork the parent steps, extends and (reset) prefills bit-identically to a run without the fork, and the
    branches give the same bits whether or not the parent advanced in between."""
    dev = _dev()
    D, t0, rows = 64, 1500, [0, 0, 1]
    op, _ = _make(D, 2000, order=3)
    up = O.nucleotide_activations(2, 1900, D)[0].to(dev)
    ub = O.nucleotide_activations(3, 100, D, seed=5)[0].to(dev)
    sched = [("step", 2), ("extend", 20), ("fft", 9), ("step", 3)]

    def parent_run(cache):
        with torch.no_grad():
            ys = [op.step(up[:, t0:t0 + 1], cache), op.extend(up[:, t0 + 1:t0 + 40], cache)]
            cache.t = 0                                   # a new sequence into the same buffers
            ys.append(op.prefill(up[:, :700], cache))
            ys.append(op.step(up[:, 700:701], cache))
        return ys

    ca, br_a = _forked(op, up.cpu(), t0, rows, 256, 2000)
    ya = parent_run(ca)                                   # the parent advances and is overwritten ...
    yb_after = _drive(op, br_a, ub, sched)                # ... before the branch runs
    cc = op.allocate_decode_cache(2, 2000)
    with torch.no_grad():
        op.prefill(up[:, :t0], cc)
    assert all(torch.equal(p, q) for p, q in zip(ya, parent_run(cc)))
    _, br_b = _forked(op, up.cpu(), t0, rows, 256, 2000)
    assert torch.equal(_drive(op, br_b, ub, sched), yb_after)


def test_select_reorder_duplicate_prune():
    dev = _dev()
    D, t0, rows = 32, 1030, [0, 0, 0, 1]
    op, P = _make(D, 1400)
    up, ub, seq = _inputs(2, t0, rows, 120, D)
    ub = ub.to(dev)
    _, br = _forked(op, up, t0, rows, 128, 1400)
    y0 = _drive(op, br, ub[:, :10], [("step", 4), ("extend", 6)])
    index = [2, 2, 0, 3]                                  # reorder, duplicate branch 2, drop branch 1
    sel = br.select(index)
    assert sel.f is br.f and sel.batch_size == 4 and sel.t == br.t
    # the same rows continuing unselected: steps give the same bits
    ya = _drive(op, br, ub[:, 10:30], [("step", 20)])
    ys = _drive(op, sel, ub[index, 10:30], [("step", 20)])
    for i, r in enumerate(index):
        assert torch.equal(ys[i], ya[r])
    # then extends on the selected rows against the truth of their sequences
    sched = [("extend", 40), ("fft", 30), ("step", 2)]
    ye = _drive(op, sel, ub[index, 30:102], sched)
    y_sel = torch.cat([y0[index].cpu(), ys.cpu(), ye.cpu()], dim=1)
    _check(y_sel, seq[index], t0, [("select", 10), ("select steps", 20)] + sched, P, "select")


def _golden_backbone(case):
    H = _H()
    z = np.load(os.path.join(GOLD, case + ".npz"))
    B, L, D, with_mlp = (int(v) for v in z["meta"])
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=2 * D, activation=partial(F.gelu, approximate="tanh")) if with_mlp else None
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return m.to(_dev()), z, B, L


@pytest.mark.parametrize("case", ["block_L128_D32_mlp", "block_L96_D16_nomlp"])
def test_backbone_golden_forked(case):
    """Fork the golden backbones after a prefill, two branches per row continuing it, driven through
    ``inference_params`` (steps and extends) and through Backbone.step / extend alike."""
    H = _H()
    m, z, B, L = _golden_backbone(case)
    x = torch.from_numpy(z["x"]).to(_dev())
    t0 = 37
    rows = [r for r in range(B) for _ in range(2)]

    def via_kwargs(xs, cache):
        h, r = xs, None
        for layer in m.layers:
            h, r = layer(h, r, mixer_kwargs={"inference_params": cache})
        return H.Block._add_norm(h, r, m.ln_f)[0]

    cache = m.allocate_decode_cache(B, L)
    with torch.no_grad():
        m.prefill(x[:, :t0], cache)
        br1, br2 = cache.fork(rows, L), cache.fork(rows, L)
        xb = x[rows]
        sched = [(1, "step"), (5, "extend"), (1, "step"), (L - t0 - 7, "extend")]
        a, b, t = [], [], t0
        for n, how in sched:
            a.append(via_kwargs(xb[:, t:t + n], br1))
            b.append(getattr(m, how)(xb[:, t:t + n], br2))
            t += n
    assert br1.branched and br1.t == L
    ya, yb = torch.cat(a, 1), torch.cat(b, 1)
    assert torch.equal(ya, yb)
    PU.check(ya.cpu(), torch.from_numpy(z["y"])[rows, t0:], f"{case} forked decode y",
             ref64=torch.from_numpy(z["y64"])[rows, t0:])


def test_launch_counts_do_not_depend_on_the_context():
    """A branch step launches the dot kernel and the branch combine per recurrence (under decode_win_step), a direct branch
    extend one hist, and one dot and one combine per recurrence; partials and grids follow H, not t0."""
    H = _H()
    lib = H._lib.lib()
    D, t0, R, horizon = 64, 9001, 5, 64
    op, _ = _make(D, 10000, order=3)
    up = O.nucleotide_activations(1, t0, D)[0]
    _, br = _forked(op, up, t0, [0] * R, horizon, 10000)
    W = br.h.shape[-1]
    assert (br.base, br.hc, W) == (9000, 64, 64)
    assert tuple(br.part.shape) == (R, D, 1)                         # ceil(H / 1024) partials, not ceil(t0 / 1024) = 9
    ub = O.nucleotide_activations(R, 20, D, seed=3)[0].to(_dev())
    with torch.no_grad():
        H._lib.profile_begin()
        op.step(ub[:, :1], br)
        prof = H._lib.profile_end()
        assert set(prof) == {"decode_win_step"} and prof["decode_win_step"][1] == 2 * 2
        j, n = br.t - br.base, 8
        groups = lib.hyena_b200_decode_extend_groups(R, D, j, n)
        assert groups == 1 and lib.hyena_b200_decode_extend_groups(R, D, br.t, n) > 1
        H._lib.profile_begin()
        op.extend(ub[:, 1:1 + n], br)
        prof = H._lib.profile_end()
        decode = {k: v[1] for k, v in prof.items() if not k.startswith("proj")}      # in_proj / out_proj GEMMs aside
        assert decode == {"decode_extend_hist": 1, "decode_extend_dot": 2, "decode_extend_combine": 2}
        n0 = H.launch_count()
        op.step(ub[:, 9:10], br)
        assert H.launch_count() - n0 == 4


def test_branches_are_deterministic():
    D, t0, rows = 64, 2003, [0, 1, 1, 0, 0]
    op, _ = _make(D, 2600)
    up = O.nucleotide_activations(2, t0, D)[0]
    ub = O.nucleotide_activations(5, 300, D, seed=9)[0].to(_dev())
    sched = [("step", 10), ("extend", 30), ("fft", 200), ("step", 5), ("direct", 55)]
    runs = [_drive(op, _forked(op, up, t0, rows, 512, 2600)[1], ub, sched) for _ in range(2)]
    assert torch.equal(runs[0], runs[1])


def test_full_length_fork():
    """D = 256, l_max = 2^20: fork 16 branches at t0 = 2^20 - 4096 + 3, then steps and extends on both routes up to Lcap.
    Every position of two branches is checked against the oracle on prefix || suffix at 2^20 (fp32 and fp64, on the GPU)."""
    dev = _dev()
    L, D, R = 1 << 20, 256, 16
    t0 = L - 4096 + 3
    op, P = _make(D, L)
    up = O.nucleotide_activations(1, t0, D)[0]
    ub = O.nucleotide_activations(R, L - t0, D, seed=11)[0]
    cache, br = _forked(op, up, t0, [0] * R, 4096, L)
    del cache
    torch.cuda.empty_cache()
    assert (br.base, br.hc) == (L - 4096, 4096)
    sched = [("step", 5), ("extend", 60), ("fft", 1000), ("step", 3), ("extend", 3025)]
    y = _drive(op, br, ub.to(dev), sched).cpu()
    assert br.t == L
    del br
    torch.cuda.empty_cache()
    P32 = {k: v.to(dev) for k, v in P.items()}
    P64 = {k: v.to(dev, torch.float64) for k, v in P.items()}
    for i in (0, 13):
        seq = torch.cat([up[0], ub[i]], dim=0)[None].to(dev)
        with torch.no_grad():
            y32 = O.hyena_operator(seq, P32)[:, t0:].cpu()                   # the reference's fp32 path (FFT), on the GPU
            y64 = O.hyena_operator(seq.double(), P64)[:, t0:].cpu()          # the oracle's fp64 truth
        torch.cuda.empty_cache()
        PU.check(y[i:i + 1], y32, f"branch {i} at L = 2^20", ref64=y64)
