"""The decoding kernels' dispatch paths against fp64.

The host code of incremental decoding (csrc/k_decode.cu, csrc/k_decode_extend.cu, csrc/api.cu) picks a kernel
instantiation, a grid and a work split from the batch size, the width, the position and the chunk length.  Each test
below drives one family of those decisions on purpose and compares every output with the fp64 oracle through
tests/parity_util.check:

| decision                               | selected by                                    | test                                  |
|----------------------------------------|------------------------------------------------|---------------------------------------|
| decode_dot_kernel<BG, R>               | BG from B (1, 2, 4, 8); R = (ld-1-t) mod 4     | test_width_batch_sweep (all 16 pairs; |
|                                        |                                                | BG 4 and 8 with a partial last group, |
|                                        |                                                | B = 9, 17: more than one z group)     |
| dot / combine channel tail             | D mod 8 (8 warps per CTA)                      | test_width_batch_sweep: D mod 8 in    |
|                                        |                                                | {1, 3, 4, 5, 6, 7}, D = 1             |
| reduce_partials lane chains            | nchunk > 32                                    | test_group_extremes[D5_t33k]          |
| decode_ext_dot_kernel<BG, NT>          | NT 8 (n <= 8, 8-warp column reduction) / 64;   | test_width_batch_sweep (all 8 pairs,  |
|                                        | R = (-t) mod 4                                 | n in 1 2 7 8 9 63 64 65)              |
| extend group count                     | hyena_b200_decode_extend_groups(B, D, t, n)    | test_group_extremes: groups = 1 with  |
|                                        |                                                | chunks per CTA > 1 (D1024), groups =  |
|                                        |                                                | nchunk (D1_t128k), causal early break |
| extend route                           | EXTEND_FFT_MIN_N                               | test_width_batch_sweep: n = 511, 512  |
| hist / ext-hist tail threads           | O + 1 channel groups                           | test_width_batch_sweep (order 2),     |
|                                        |                                                | test_orders (3, 4) at D = 23, 100     |
| Lcap mod 4                             | ld_for padding of the reversed filter          | every case; 0, 1, 2 and 3 all hit     |
| B * D > 65535                          | launch_decode_hist grid (rows on x)            | test_large_batch, test_large_batch_   |
|                                        |                                                | backbone_and_ragged                   |

Beyond the table: windowed steps, forks with 3 to 17 branches and select, StepGraph replays and ragged prefill at tail
widths (test_windowed_steps_tail_widths, test_fork_select_tail_widths, test_step_graph_tail_widths,
test_ragged_prefill_tail_width); a two-layer Backbone with Mlp at D = 3 and 100 against an fp64 composition of its own
parameters (test_backbone_decoding_tail_widths); and row isolation: a NaN or +-inf batch row, branch or pad stays out of
the other rows (test_operator_row_isolation, test_kernel_rows_bitwise, test_branch_isolation, and the fills of
tests/test_gpu_ragged.py's pad-independence tests).

Every GPU case also reads the library's profiler to confirm that the route it targets ran.  The fp32 twin of the reference
is passed as ``ref32`` and its fp64 truth as ``ref64``, so any use of the S8(c) hatch is book-kept.  The tests marked
``gpu`` need an H100; the self-checks of the references, of the bar and of the coverage table run on the CPU.
"""
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_gpu_widths import NANS, _poison

gpu = pytest.mark.gpu

KCHUNK = 1024            # positions per partial of the dot kernels (csrc/decode_args.h kChunk)
FFT_MIN_N = 512          # ops.EXTEND_FFT_MIN_N (pinned by test_coverage_table)


# ------------------------------------------------------------------------------------------ the cases
def sweep_schedule(P0):
    """Prefill, steps over every t mod 4 across the 1024-position chunk boundary (P0 ~ 1020), direct extends of every
    tile shape and tail, both sides of the FFT threshold, more steps."""
    return [("prefill", P0), ("step", 6), ("direct", 1), ("direct", 2), ("direct", 7), ("direct", 8), ("direct", 9),
            ("direct", 63), ("direct", 64), ("direct", 65), ("direct", FFT_MIN_N - 1), ("fft", FFT_MIN_N), ("step", 5)]


# (D, B, P0): every D mod 8 tail with a batch that gives each batch group a tail; P0 sets Lcap = P0 + 1253 to 1, 2, 3 mod 4
SWEEP = [(1, 17, 1020), (3, 9, 1021), (5, 5, 1022), (14, 3, 1020), (23, 2, 1021), (100, 1, 1022), (1020, 8, 1021)]
# (D, B, order, P0)
ORDERS = [(23, 3, 3, 1019), (100, 2, 3, 1020), (23, 2, 4, 1022), (100, 3, 4, 1019)]
# name -> (D, B, schedule): long histories and the extremes of the extend group count, checked at the decoded positions
LONG = {
    "D1_t128k": (1, 1, [("prefill", (1 << 17) - 5), ("step", 5), ("direct", 9), ("direct", 64), ("step", 2)]),
    "D1024_groups1": (1024, 17, [("prefill", 1980), ("direct", 100), ("step", 2)]),
    "D5_t33k": (5, 3, [("prefill", 33 * KCHUNK + 1), ("step", 6), ("direct", 3)]),
}
# (D, B, schedule) at B * D > 65535
LARGE = [(256, 257, [("prefill", 37), ("step", 3), ("direct", 9)]), (1024, 65, [("prefill", 21), ("step", 2), ("direct", 5)])]


def sched_len(sched):
    return sum(n for _, n in sched)


# ------------------------------------------------------------------------------------------ fp64 references
def direct_ref(u, P, pos, dtype, dev, conv=None):
    """Order-2 outputs at positions ``pos`` by direct dot products over the history, in ``dtype`` on ``dev``:
    y[t] = out_proj((sum_{s<=t} k[t-s] g[s] + bias g[t]) x0[t]).  With ``conv`` (e.g. O.fftconv_direct) the whole
    convolution is taken from it instead (the self-check)."""
    Q = {k: v.to(dev, dtype) for k, v in P.items()}
    B, L, D = u.shape
    p = F.linear(u.to(dev, dtype), Q["in_proj.weight"], Q["in_proj.bias"]).transpose(1, 2)
    uc = O.short_filter(p, Q["short_filter.weight"], Q["short_filter.bias"], L)
    del p
    x0, x1, v = uc.split(D, dim=1)
    g = (v * x1).contiguous()
    k = O.hyena_filter(L, Q)[0].transpose(0, 1)                                # (D, L)
    if conv is not None:
        c = conv(g, k, Q["filter_fn.bias"])[:, :, pos]
    else:
        c = torch.stack([(g[:, :, :t + 1] * k[:, :t + 1].flip(-1)).sum(-1) + Q["filter_fn.bias"] * g[:, :, t] for t in pos],
                        dim=-1)
    y_pre = (c * x0[:, :, pos]).transpose(1, 2)                                 # (B, len(pos), D)
    return F.linear(y_pre, Q["out_proj.weight"], Q["out_proj.bias"])


def backbone_ref(x, sd, n_layer, dtype, eps=1e-5, fp32_residual=False):
    """A pre-norm Backbone composed in ``dtype`` from a state_dict: per block add -> LayerNorm -> oracle operator -> add ->
    LayerNorm -> fc2(gelu_tanh(fc1(.))), then add -> ln_f.  The residual stream stays in ``dtype``; ``fp32_residual``
    rounds it to fp32 after each LayerNorm, as the reference Block does with residual_in_fp32 (its fp64 golden run)."""
    rnd = (lambda r: r.float().to(dtype)) if fp32_residual else (lambda r: r)
    S = {k: v.to(x.device, dtype) for k, v in sd.items()}
    D = x.shape[-1]
    hidden, residual = x.to(dtype), None
    for i in range(n_layer):
        pre = f"layers.{i}."
        residual = hidden + residual if residual is not None else hidden
        h = F.layer_norm(residual, (D,), S[pre + "norm1.weight"], S[pre + "norm1.bias"], eps)
        residual = rnd(residual)
        P = O.canonical({k[len(pre + "mixer."):]: v for k, v in S.items() if k.startswith(pre + "mixer.")})
        hidden = O.hyena_operator(h, P)
        if pre + "mlp.fc1.weight" in S:
            residual = hidden + residual
            h = F.layer_norm(residual, (D,), S[pre + "norm2.weight"], S[pre + "norm2.bias"], eps)
            residual = rnd(residual)
            h = F.gelu(F.linear(h, S[pre + "mlp.fc1.weight"], S[pre + "mlp.fc1.bias"]), approximate="tanh")
            hidden = F.linear(h, S[pre + "mlp.fc2.weight"], S[pre + "mlp.fc2.bias"])
    return F.layer_norm(hidden + residual, (D,), S["ln_f.weight"], S["ln_f.bias"], eps)


def _params(D, L, order=2, seed=0):
    """Oracle parameters with a non-zero in_proj bias (the decode kernels add it themselves)."""
    g = torch.Generator().manual_seed(seed)
    P = O.init_params(D, L, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    P["in_proj.bias"] = 0.02 * torch.randn(P["in_proj.bias"].shape, generator=g)
    return P


def _input(B, L, D, seed=2222):
    """The nucleotide activation of the benchmark; at D = 1, where its LayerNorm gives all zeros, a normal input."""
    if D == 1:
        return torch.randn(B, L, D, generator=torch.Generator().manual_seed(seed))
    return O.nucleotide_activations(B, L, D, seed=seed)[0]


# ------------------------------------------------------------------------------------------ CPU self-checks
@pytest.mark.parametrize("B,L,D", [(2, 37, 3), (3, 70, 1)])
def test_direct_ref_matches_oracle_and_direct_convolution(B, L, D):
    P = O.to_dtype(_params(D, L, seed=L), torch.float64)
    u = _input(B, L, D, seed=L).double()
    pos = list(range(L))
    y = direct_ref(u, P, pos, torch.float64, "cpu")
    torch.testing.assert_close(y, O.hyena_operator(u, P), rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(y, direct_ref(u, P, pos, torch.float64, "cpu", conv=O.fftconv_direct), rtol=1e-10,
                               atol=1e-12)
    sub = [0, 5, L - 1]
    torch.testing.assert_close(direct_ref(u, P, sub, torch.float64, "cpu"), y[:, sub], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("case", ["block_L128_D32_mlp", "block_L96_D16_nomlp"])
def test_backbone_ref_matches_golden(case):
    """backbone_ref in fp64 gives the fp64 output of the reference's own Block + Mlp stack (tests/golden), and without
    the fp32 residual rounding stays within 1e-6 of it."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", case + ".npz"))
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
    y = backbone_ref(torch.from_numpy(z["x"]), sd, 2, torch.float64, fp32_residual=True)
    torch.testing.assert_close(y, torch.from_numpy(z["y64"]), rtol=1e-9, atol=1e-9)
    torch.testing.assert_close(backbone_ref(torch.from_numpy(z["x"]), sd, 2, torch.float64), y, rtol=0, atol=1e-6)


def _decode_parts(u, P):
    """fp64 pieces of the order-2 operator: g, k, bias, x0 (B, D, L) and the convolution c by the O(L^2) sum."""
    B, L, D = u.shape
    p = F.linear(u, P["in_proj.weight"], P["in_proj.bias"]).transpose(1, 2)
    uc = O.short_filter(p, P["short_filter.weight"], P["short_filter.bias"], L)
    x0, x1, v = uc.split(D, dim=1)
    g = v * x1
    k = O.hyena_filter(L, P)[0].transpose(0, 1)
    return g, k, P["filter_fn.bias"], x0, O.fftconv_direct(g, k, P["filter_fn.bias"])


def _tap(g, k, t, shift):
    """sum_{s<=t} k[t-s+shift] g[s] at one position (k zero outside [0, L))."""
    L = k.shape[-1]
    s = torch.arange(t + 1)
    idx = t - s + shift
    ok = (idx >= 0) & (idx < L)
    return (g[:, :, s[ok]] * k[:, idx[ok]]).sum(-1)


BUGS = ["tail channels take channel d-1's filter", "row 8 adds row 0's history", "last partial chunk dropped",
        "filter read one tap off at one residue", "tile output j takes column j+1's taps", "bias g[t] dropped at one position"]


@pytest.mark.parametrize("bug", BUGS)
def test_parity_bar_rejects_decode_bugs(bug):
    """The bar can tell a correct decode from one with a bug these paths could have: each bug is applied to the fp64
    truth, which must then be rejected against the fp32 / fp64 pair that the unperturbed truth passes."""
    B, D, L, t0 = 9, 13, 1100, 1030                     # D mod 8 = 5; positions [t0, L) decoded, past a chunk boundary
    P = _params(D, L, seed=7)
    u = _input(B, L, D, seed=7)
    y32 = O.hyena_operator(u, P)[:, t0:]
    P64 = O.to_dtype(P, torch.float64)
    g, k, fb, x0, c = _decode_parts(u.double(), P64)
    y64 = F.linear((c * x0).transpose(1, 2), P64["out_proj.weight"], P64["out_proj.bias"])[:, t0:]
    c = c.clone()
    if bug == BUGS[0]:
        tail = D - D % 8
        kw = k.clone()
        kw[tail:] = k[tail - 1:D - 1]
        c[:, tail:] = O.fftconv_direct(g[:, tail:], kw[tail:], fb[tail:])[:, :, :]
    elif bug == BUGS[1]:
        c[8] += O.fftconv_direct(g[0:1], k, torch.zeros_like(fb))[0]
    elif bug == BUGS[2]:
        t = L - 1
        s0 = t // KCHUNK * KCHUNK
        c[:, :, t] -= (g[:, :, s0:t] * k[:, 1:t - s0 + 1].flip(-1)).sum(-1)
    elif bug == BUGS[3]:
        for t in range(t0 + 1, L, 4):
            c[:, :, t] = _tap(g, k, t, 1) + fb * g[:, :, t]
    elif bug == BUGS[4]:
        t = t0 + 3
        c[:, :, t] = _tap(g, k, t, 1) + fb * g[:, :, t]
    elif bug == BUGS[5]:
        t = t0 + 5
        c[:, :, t] -= fb * g[:, :, t]
    wrong = F.linear((c * x0).transpose(1, 2), P64["out_proj.weight"], P64["out_proj.bias"])[:, t0:]
    n0 = len(PU._records)
    try:
        PU.check(y64.float(), y32, "unperturbed", ref64=y64)
        with pytest.raises(AssertionError):
            PU.check(wrong, y32, bug, ref64=y64)
    finally:
        del PU._records[n0:]            # self-checks of the bar, not parity records


def _groups_lib():
    import hyena_dna_b200 as H
    return H._lib.lib().hyena_b200_decode_extend_groups


def _bg(B):
    return 1 if B <= 1 else 2 if B <= 2 else 4 if B <= 4 else 8


def decisions(B, D, order, sched, lcap, groups_fn):
    """The host decisions a schedule takes (csrc/k_decode.cu launch_dot, k_decode_extend.cu, decode_args.h), as a set of
    tuples, computed from the shapes alone."""
    ld = (lcap + 3) // 4 * 4
    hit = {("lcap mod 4", lcap % 4), ("order", order, D % 8 != 0)}
    t = 0
    for how, n in sched:
        if how == "prefill":
            hit.add(("hist", B * D > 65535))
            t += n
            continue
        if how == "step":
            for s in range(t, t + n):
                if s > 0:
                    nchunk = -(-s // KCHUNK)
                    hit |= {("dot", _bg(B), (ld - 1 - s) % 4), ("tail", D % 8), ("dot z groups", _bg(B), -(-B // _bg(B)))}
                    hit.add(("partial group", _bg(B), B % _bg(B) != 0))
                    if nchunk > 32:
                        hit.add(("lane chains", D % 8 != 0))
            t += n
            continue
        fft = how == "fft" or (how == "extend" and n >= FFT_MIN_N)
        hit.add(("route", n, fft, D % 8 != 0))
        if not fft:
            NT = 8 if n <= 8 else 64
            hit |= {("ext", _bg(B), NT), ("ext n", n), ("ext R", NT, (-t) % 4)}
            nchunk = -(-(t + n) // KCHUNK)
            groups = groups_fn(B, D, t, n)
            cpb = -(-nchunk // groups)
            if groups == 1 and cpb > 1:
                hit.add(("groups", "one group, several chunks"))
            if groups == nchunk:
                hit.add(("groups", "one group per chunk"))
            for g in range(groups):
                for j0 in range(0, n, NT):
                    if any(c * KCHUNK > t + j0 + NT - 1 for c in range(g * cpb, min((g + 1) * cpb, nchunk))):
                        hit.add(("groups", "causal break"))
        t += n
    return hit


def all_cases():
    """(B, D, order, schedule, Lcap) of every operator-level case of the file that the table counts."""
    out = [(B, D, 2, sweep_schedule(P0), sched_len(sweep_schedule(P0))) for D, B, P0 in SWEEP]
    out += [(B, D, order, sweep_schedule(P0), sched_len(sweep_schedule(P0))) for D, B, order, P0 in ORDERS]
    out += [(B, D, 2, s, sched_len(s)) for D, B, s in LONG.values()]
    out += [(B, D, 2, s, sched_len(s)) for D, B, s in LARGE]
    return out


def test_coverage_table():
    """Every cell of the module docstring's table is hit by the cases above; the group counts come from the library."""
    import hyena_dna_b200 as H
    assert H.ops.EXTEND_FFT_MIN_N == FFT_MIN_N
    groups = _groups_lib()
    hit = set()
    for B, D, order, sched, lcap in all_cases():
        hit |= decisions(B, D, order, sched, lcap, groups)
    want = {("dot", bg, r) for bg in (1, 2, 4, 8) for r in range(4)}
    want |= {("partial group", 4, True), ("partial group", 8, True), ("dot z groups", 8, 2), ("dot z groups", 8, 3)}
    want |= {("tail", r) for r in (1, 3, 4, 5, 6, 7)} | {("lane chains", True)}
    want |= {("ext", bg, nt) for bg in (1, 2, 4, 8) for nt in (8, 64)}
    want |= {("ext n", n) for n in (1, 2, 7, 8, 9, 63, 64, 65)}
    want |= {("ext R", nt, r) for nt in (8, 64) for r in range(4)}
    want |= {("groups", "one group, several chunks"), ("groups", "one group per chunk"), ("groups", "causal break")}
    want |= {("route", FFT_MIN_N - 1, False, True), ("route", FFT_MIN_N, True, True)}
    want |= {("order", o, True) for o in (2, 3, 4)}
    want |= {("lcap mod 4", r) for r in range(4)} | {("hist", True)}
    assert not want - hit, f"table cells not hit: {sorted(want - hit, key=str)}"
    assert any(D == 1 for _, D, *_ in all_cases())
    # the two group extremes are the cases named for them
    D, B, s = LONG["D1024_groups1"]
    t, n = s[0][1], s[1][1]
    assert groups(B, D, t, n) == 1 and -(-(t + n) // KCHUNK) > 1
    D, B, s = LONG["D1_t128k"]
    t = s[0][1] + s[1][1]
    assert groups(B, D, t, 9) == -(-(t + 9) // KCHUNK)


# ------------------------------------------------------------------------------------------ device helpers
def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _operator(P, D, L, order=2):
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = _H().HyenaOperator(D, L, order=order, emb_dim=5, w=10.0)
    op.load_state_dict(sd)
    return op.to(_dev())


def _truth(u, P, dev):
    """The oracle on the device: fp32 (TF32 off) and fp64."""
    P32 = {k: v.to(dev) for k, v in P.items()}
    with torch.no_grad():
        y32 = O.hyena_operator(u.to(dev), P32)
        y64 = O.hyena_operator(u.to(dev, torch.float64), O.to_dtype(P32, torch.float64))
    return y32, y64


def _route_ok(how, prof, nrec, window=False):
    """The profiler window of one schedule entry shows the route it targets."""
    if how == "prefill":
        assert "decode_hist" in prof, prof
    elif how == "step":
        assert ("decode_win_step" if window else "decode_step") in prof, prof
    elif how == "direct":
        assert prof.get("decode_extend_dot", (0, 0))[1] == nrec, prof
    elif how == "fft":
        assert "decode_extend_dot" not in prof and prof.get("decode_extend_combine", (0, 0))[1] == nrec, prof
    elif how == "extend":
        assert "decode_extend_combine" in prof, prof


def _run(m, u, sched, cache, nrec=1, window=False):
    """Feed u (on the GPU) to m from cache.t on by the schedule [(how, n), ...]: prefill, step, extend (the route rule),
    direct / fft (an operator's extend forced onto that route); each entry's route is confirmed by the profiler."""
    H = _H()
    outs, t = [], cache.t
    with torch.no_grad():
        for how, n in sched:
            H._lib.profile_begin()
            if how == "step":
                outs += [m.step(u[:, s:s + 1], cache) for s in range(t, t + n)]
            elif how in ("direct", "fft"):
                core = H.ops.decode_extend_direct if how == "direct" else H.ops.decode_extend_fft
                if cache.branched:
                    core = partial(H.ops.decode_branch_extend, fft=how == "fft")
                outs.append(m._extend(u[:, t:t + n], cache.for_module(m), core))
            else:
                outs.append(getattr(m, how)(u[:, t:t + n], cache))
            _route_ok(how, H._lib.profile_end(), nrec, window and how == "step")
            t += n
    assert cache.t == t
    return torch.cat(outs, dim=1)


def _check_chunks(y, y32, y64, sched, what, t0=0):
    t = 0
    for how, n in sched:
        if how != "prefill" or t0 == 0:
            PU.check(y[:, t:t + n], y32[:, t:t + n], f"{what} {how} [{t0 + t}, {t0 + t + n})", ref64=y64[:, t:t + n])
        t += n


def _operator_case(D, B, order, sched, what, seed):
    dev = _dev()
    L = sched_len(sched)
    P = _params(D, L, order, seed)
    op = _operator(P, D, L, order)
    u = _input(B, L, D, seed)
    cache = op.allocate_decode_cache(B, L)
    assert cache.lcap == L
    y = _run(op, u.to(dev), sched, cache, nrec=order - 1)
    y32, y64 = _truth(u, P, dev)
    _check_chunks(y, y32, y64, sched, what)


# ------------------------------------------------------------------------------------------ 1. width x batch sweep
@gpu
@pytest.mark.parametrize("D,B,P0", SWEEP)
def test_width_batch_sweep(D, B, P0):
    _operator_case(D, B, 2, sweep_schedule(P0), f"sweep D={D} B={B}", seed=D * 31 + B)


# ------------------------------------------------------------------------------------------ 2. orders 3 and 4
@gpu
@pytest.mark.parametrize("D,B,order,P0", ORDERS)
def test_orders(D, B, order, P0):
    _operator_case(D, B, order, sweep_schedule(P0), f"order {order} D={D} B={B}", seed=order * 100 + D)


# ------------------------------------------------------------------------------------------ 3. group extremes, long histories
@gpu
@pytest.mark.parametrize("name", list(LONG))
def test_group_extremes(name):
    """After the prefill, every decoded position against fp64 direct dot products over the whole history."""
    dev = _dev()
    D, B, sched = LONG[name]
    L, t0 = sched_len(sched), sched[0][1]
    P = _params(D, L, seed=len(name))
    op = _operator(P, D, L)
    u = _input(B, L, D, seed=len(name))
    cache = op.allocate_decode_cache(B, L)
    y = _run(op, u.to(dev), sched, cache)[:, t0:]
    pos = list(range(t0, L))
    with torch.no_grad():
        y64 = direct_ref(u, P, pos, torch.float64, dev)
        y32 = direct_ref(u, P, pos, torch.float32, dev)
    _check_chunks(y, y32, y64, sched[1:], f"long {name}", t0=t0)


@gpu
def test_unaligned_single_sequence_views():
    """B = 1 at D = 3: forward, prefill, steps and extends of views that start 12 bytes into a 16-byte word (u[:, 1:] and
    its slices at odd t) against fp64.  The projection GEMM copies such operands to an aligned allocation; before, the
    extend of a D = 1 sequence at t = 2^17 raised "pointers must be 16-byte aligned"."""
    dev = _dev()
    B, D, L = 1, 3, 300
    P = _params(D, L + 1, seed=3)
    op = _operator(P, D, L + 1)
    u = _input(B, L + 1, D, seed=3)
    ud = u.to(dev)[:, 1:]
    assert ud.is_contiguous() and ud.data_ptr() % 16 == 12
    y32, y64 = _truth(u[:, 1:], P, dev)
    with torch.no_grad():
        PU.check(op(ud), y32, "forward of an unaligned view", ref64=y64)
    sched = [("prefill", 101), ("direct", 7), ("step", 1), ("extend", 9), ("fft", 182)]
    y = _run(op, ud, sched, op.allocate_decode_cache(B, L))
    _check_chunks(y, y32, y64, sched, "unaligned views")


# ------------------------------------------------------------------------------------------ 4. windows, forks, graphs, ragged
@pytest.fixture
def small_windows(monkeypatch):
    """Windows of 64 positions that open after 2 steps at any history."""
    ops = _H().ops
    monkeypatch.setattr(ops, "WINDOW", 64)
    monkeypatch.setattr(ops, "WINDOW_MIN_T", 0)
    monkeypatch.setattr(ops, "WINDOW_AFTER_STEPS", 2)


@gpu
@pytest.mark.parametrize("D,B,P0", [(100, 5, 1021), (3, 9, 998), (23, 17, 1)])
def test_windowed_steps_tail_widths(small_windows, D, B, P0):
    """Two plain steps, then windowed steps over more than three windows (every t mod 4, window bases on both sides of a
    1024-position chunk boundary), an extend inside the open window, and windowed steps again."""
    dev = _dev()
    sched = [("prefill", P0), ("step", 2), ("wstep", 3 * 64 + 41), ("direct", 9), ("wstep", 9)]
    L = sched_len(sched)
    P = _params(D, L, seed=D + B)
    op = _operator(P, D, L)
    u = _input(B, L, D, seed=D + B)
    cache = op.allocate_decode_cache(B, L)
    y = torch.cat([_run(op, u.to(dev), [(how.lstrip("w"), n)], cache, window=how == "wstep") for how, n in sched], dim=1)
    assert cache.win_wc > 0
    y32, y64 = _truth(u, P, dev)
    _check_chunks(y, y32, y64, sched, f"window D={D} B={B}")


def _branch_drive(op, br, seq, sched):
    """Branch steps (counted as windowed steps) and extends; seq (R, >= t, D) holds each branch's whole sequence."""
    return _run(op, seq, sched, br, window=True)


FORKS = [(23, 2, 1021, [1, 0, 1]), (100, 3, 1022, [2, 2, 0, 1, 2]), (3, 2, 1023, [0, 1, 1, 0, 0, 1, 0, 1, 1]),
         (5, 4, 1024, [3, 0, 0, 1, 2, 3, 3, 1, 0, 2, 2, 1, 0, 3, 1, 2, 0])]


@gpu
@pytest.mark.parametrize("D,B,t0,rows", FORKS)
def test_fork_select_tail_widths(D, B, t0, rows):
    """R = 3, 5, 9, 17 branches with repeated and mixed parents at t0 of every residue mod 4: branch steps and both
    extend routes, then select (reordered with repeats) and more of both, against the oracle on prefix || branch."""
    dev = _dev()
    R = len(rows)
    s1 = [("step", 2), ("direct", 7), ("step", 1), ("fft", 9), ("direct", 3)]
    s2 = [("step", 3), ("direct", 5), ("fft", 4), ("step", 1)]
    m1, m2 = sched_len(s1), sched_len(s2)
    lcap = t0 + m1 + m2 + 64
    P = _params(D, lcap, seed=R)
    op = _operator(P, D, lcap)
    up = _input(B, t0, D, seed=R)
    ub = _input(R, m1 + m2, D, seed=R + 1)
    cache = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(up.to(dev), cache)
    br = cache.fork(rows, horizon=64)
    seq1 = torch.cat([up[rows], ub[:, :m1]], dim=1)
    y1 = _branch_drive(op, br, seq1.to(dev), s1)
    y32, y64 = _truth(seq1, P, dev)
    _check_chunks(y1, y32[:, t0:], y64[:, t0:], s1, f"fork D={D} R={R}", t0=t0)
    idx = [(3 * i + 1) % R for i in range(R)]
    sel = br.select(idx)
    seq2 = torch.cat([seq1[idx], ub[idx, m1:]], dim=1)
    y2 = _branch_drive(op, sel, seq2.to(dev), s2)
    y32, y64 = _truth(seq2, P, dev)
    _check_chunks(y2, y32[:, t0 + m1:], y64[:, t0 + m1:], s2, f"select D={D} R={R}", t0=t0 + m1)


@gpu
@pytest.mark.parametrize("D,B", [(100, 5), (3, 9)])
def test_step_graph_tail_widths(D, B):
    """StepGraph replays across the 1024-position chunk boundary are the bits of eager steps on a twin cache, and both
    pass the bar against fp64."""
    H = _H()
    dev = _dev()
    P0, n = 1019, 9
    L = P0 + n
    P = _params(D, L, seed=D)
    op = _operator(P, D, L)
    u = _input(B, L, D, seed=D)
    ud = u.to(dev)
    ce, cg = op.allocate_decode_cache(B, L), op.allocate_decode_cache(B, L)
    with torch.no_grad():
        op.prefill(ud[:, :P0], ce)
        op.prefill(ud[:, :P0], cg)
    g = H.StepGraph(op, cg, B, torch.float32)
    ys = []
    with torch.no_grad():
        for i in range(P0, L):
            ye, yg = op.step(ud[:, i:i + 1], ce), g.step(ud[:, i:i + 1])
            assert torch.equal(ye, yg), f"D={D} B={B} position {i}: graph and eager steps differ"
            ys.append(yg.clone())               # the graph's output buffer is rewritten by the next replay
    assert set(g._graphs) == {"plain"}
    y32, y64 = _truth(u, P, dev)
    PU.check(torch.cat(ys, dim=1), y32[:, P0:], f"graph D={D} B={B}", ref64=y64[:, P0:])


def _ragged_case(D, lengths, P0, cont_sched, seed, what):
    """Left-padded prefill of rows of ``lengths`` at width D, then cont_sched; each row against the oracle on its
    unpadded tokens followed by its continuation."""
    dev = _dev()
    B = len(lengths)
    m = sched_len(cont_sched)
    L = P0 + m
    P = _params(D, L, seed=seed)
    op = _operator(P, D, L)
    u = _input(B, L, D, seed=seed)
    g = torch.Generator().manual_seed(seed)
    for b, n in enumerate(lengths):
        u[b, :P0 - n] = 3.0 * torch.randn(P0 - n, D, generator=g)
    cache = op.allocate_decode_cache(B, L)
    with torch.no_grad():
        y0 = op.prefill(u[:, :P0].to(dev), cache, lengths=lengths)
    y = torch.cat([y0, _run(op, u.to(dev), cont_sched, cache)], dim=1)
    for n in sorted(set(lengths)):
        rows = [b for b, x in enumerate(lengths) if x == n]
        y32, y64 = _truth(u[rows, P0 - n:], P, dev)
        PU.check(y[rows, P0 - n:], y32, f"{what} rows of length {n}", ref64=y64)


@gpu
def test_ragged_prefill_tail_width():
    _ragged_case(100, [1030, 1, 37, 1027, 500], 1030, [("step", 5), ("direct", 9), ("step", 2)], 100, "ragged D=100")


# ------------------------------------------------------------------------------------------ 5. large batches
@gpu
@pytest.mark.parametrize("D,B,sched", LARGE, ids=["B257_D256", "B65_D1024"])
def test_large_batch(D, B, sched):
    """B * D > 65535 rows of the prefill's history kernel; then steps and an extend."""
    _operator_case(D, B, 2, sched, f"large batch D={D} B={B}", seed=B)


def _backbone(D, L, seed):
    H = _H()
    torch.manual_seed(seed)
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=4 * D, activation=partial(F.gelu, approximate="tanh"))
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.LayerNorm):
                mod.weight.add_(0.1 * torch.randn_like(mod.weight))
                mod.bias.add_(0.1 * torch.randn_like(mod.bias))
            if isinstance(mod, H.HyenaOperator):
                mod.in_proj.bias.normal_(0, 0.02)
    return m.to(_dev())


def _backbone_truth(m, x, dev):
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    with torch.no_grad():
        return backbone_ref(x.to(dev), sd, 2, torch.float32), backbone_ref(x.to(dev), sd, 2, torch.float64)


@gpu
def test_large_batch_backbone_and_ragged():
    """Backbone.prefill and a step at B = 257, D = 256 against the fp64 composition; ragged prefill and a step at the same
    size against the oracle per row length."""
    dev = _dev()
    B, D, P0 = 257, 256, 24
    m = _backbone(D, P0 + 2, seed=3)
    x = torch.randn(B, P0 + 2, D, generator=torch.Generator().manual_seed(3))
    cache = m.allocate_decode_cache(B, P0 + 2)
    sched = [("prefill", P0), ("step", 2)]
    y = _run(m, x.to(dev), sched, cache, nrec=2)
    y32, y64 = _backbone_truth(m, x, dev)
    _check_chunks(y, y32, y64, sched, "backbone B=257 D=256")
    _ragged_case(D, [P0, 1, 17, 9] * 64 + [P0], P0, [("step", 2), ("direct", 3)], 257, "ragged B=257 D=256")


# ------------------------------------------------------------------------------------------ 6. backbone at tail widths
@gpu
@pytest.mark.parametrize("D", [3, 100])
def test_backbone_decoding_tail_widths(D):
    """A 2-layer Backbone with Mlp: prefill, steps, an extend, steps, against an fp64 composition of its own parameters;
    StepGraph replays on a twin cache give the bits of the eager steps."""
    H = _H()
    dev = _dev()
    B, P0 = 3, 301
    sched = [("prefill", P0), ("step", 3), ("extend", 9), ("step", 4)]
    L = sched_len(sched)
    m = _backbone(D, L, seed=D)
    x = torch.randn(B, L, D, generator=torch.Generator().manual_seed(D))
    xd = x.to(dev)
    cache = m.allocate_decode_cache(B, L)
    y = _run(m, xd, sched, cache, nrec=2)
    y32, y64 = _backbone_truth(m, x, dev)
    _check_chunks(y, y32, y64, sched, f"backbone D={D}")
    cg = m.allocate_decode_cache(B, L)
    with torch.no_grad():
        m.prefill(xd[:, :P0], cg)
        g = H.StepGraph(m, cg, B, torch.float32)
        for i in range(P0, P0 + 3):
            assert torch.equal(g.step(xd[:, i:i + 1]), y[:, i:i + 1]), f"backbone D={D}: graph step {i} differs"


# ------------------------------------------------------------------------------------------ 7. row isolation
KINDS = [*NANS, "inf"]


@gpu
def test_operator_row_isolation(small_windows):
    """B = 9 at D = 100 with row 4 all NaN (three encodings) or all +-inf: prefill, plain and windowed steps, both extend
    routes.  The other rows are finite and pass the bar against the oracle on each row alone; row 4 stays non-finite."""
    dev = _dev()
    B, D, bad = 9, 100, 4
    sched = [("prefill", 300), ("step", 2), ("wstep", 5), ("direct", 9), ("fft", FFT_MIN_N), ("step", 2), ("wstep", 3)]
    L = sched_len(sched)
    P = _params(D, L, seed=9)
    op = _operator(P, D, L)
    u = _input(B, L, D, seed=9)
    truth = {b: _truth(u[b:b + 1], P, dev) for b in range(B) if b != bad}
    for kind in KINDS:
        u2 = u.clone()
        u2[bad] = _poison(u[bad], kind, torch.Generator().manual_seed(4))
        cache = op.allocate_decode_cache(B, L)
        y = torch.cat([_run(op, u2.to(dev), [(how.lstrip("w"), n)], cache, window=how == "wstep") for how, n in sched],
                      dim=1)
        assert not bool(torch.isfinite(y[bad]).any()), f"{kind}: finite outputs in the poisoned row"
        for b, (y32, y64) in truth.items():
            _check_chunks(y[b:b + 1], y32, y64, sched, f"isolation {kind} row {b}")


@gpu
def test_kernel_rows_bitwise():
    """ops.decode_hist / decode_step / decode_extend_direct at B = 9 with row 4 poisoned: every other row is bit-identical
    to the B = 1 run of that row (a row's arithmetic in these kernels does not depend on B), and row 4 is non-finite."""
    H = _H()
    ops = H.ops
    dev = _dev()
    B, D, P0, n, bad = 9, 100, 1030, 9, 4
    L = P0 + 1 + n
    P = _params(D, L, seed=11)
    op = _operator(P, D, L)
    ib, sw, sb = op._decode_params()
    gen = torch.Generator(device=dev).manual_seed(11)
    p = torch.randn(B, 3 * D, P0, generator=gen, device=dev)
    p_t = torch.randn(B, 3 * D, generator=gen, device=dev)
    pe = torch.randn(B, 3 * D, n, generator=gen, device=dev)
    groups = _groups_lib()
    same_groups = groups(B, D, P0 + 1, n) == groups(1, D, P0 + 1, n)
    assert same_groups, "this case is meant to have the same extend group count at B = 9 and at B = 1"

    def run(pp, pt, ppe, rows):
        c = op.allocate_decode_cache(rows, L)
        ops.decode_hist(pp.contiguous(), ib, sw, sb, c)
        h, tail = c.h[..., :P0].clone(), c.tail.clone()
        c.t = P0
        y = ops.decode_step(pt.contiguous(), ib, sw, sb, c)
        c.t += 1
        e = ops.decode_extend_direct(ppe.contiguous(), ib, sw, sb, c)
        return h, tail, y, e

    alone = {b: run(p[b:b + 1], p_t[b:b + 1], pe[b:b + 1], 1) for b in range(B) if b != bad}
    for kind in KINDS:
        g = torch.Generator(device=dev).manual_seed(5)
        p2, pt2, pe2 = p.clone(), p_t.clone(), pe.clone()
        p2[bad], pt2[bad], pe2[bad] = _poison(p[bad], kind, g), _poison(p_t[bad], kind, g), _poison(pe[bad], kind, g)
        h, tail, y, e = run(p2, pt2, pe2, B)
        assert not bool(torch.isfinite(y[bad]).any()) and not bool(torch.isfinite(e[bad]).any()), kind
        for b, (h1, tail1, y1, e1) in alone.items():
            assert torch.equal(h[:, b], h1[:, 0]) and torch.equal(tail[b], tail1[0]), f"{kind} row {b}: history / tail"
            assert torch.equal(y[b], y1[0]), f"{kind} row {b}: step output"
            assert torch.equal(e[b], e1[0]), f"{kind} row {b}: extend output"


@gpu
def test_branch_isolation():
    """Branches forked from a poisoned parent row leave the branches of the clean rows intact."""
    dev = _dev()
    B, D, t0, bad = 3, 23, 1022, 1
    rows = [0, bad, 2, bad, 0]
    s1 = [("step", 2), ("direct", 7), ("fft", 9), ("step", 1)]
    m1 = sched_len(s1)
    lcap = t0 + m1 + 64
    P = _params(D, lcap, seed=13)
    op = _operator(P, D, lcap)
    up = _input(B, t0, D, seed=13)
    ub = _input(len(rows), m1, D, seed=14)
    seq = torch.cat([up[rows], ub], dim=1)
    y32, y64 = _truth(seq, P, dev)
    for kind in KINDS:
        up2 = up.clone()
        up2[bad] = _poison(up[bad], kind, torch.Generator().manual_seed(6))
        cache = op.allocate_decode_cache(B, lcap)
        with torch.no_grad():
            op.prefill(up2.to(dev), cache)
        br = cache.fork(rows, horizon=64)
        y = _branch_drive(op, br, seq.to(dev), s1)
        for i, r in enumerate(rows):
            if r == bad:
                assert not bool(torch.isfinite(y[i]).any()), f"{kind}: finite outputs in branch {i} of the poisoned row"
            else:
                _check_chunks(y[i:i + 1], y32[i:i + 1, t0:], y64[i:i + 1, t0:], s1, f"branch isolation {kind} {i}", t0=t0)
