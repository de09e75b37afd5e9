"""Extending a decode cache by many positions at once (HyenaOperator / Block / Backbone extend, csrc/decode_extend.cuh)
against the fp64 truth of the oracle on the whole sequence.  Tolerance policy: tests/parity_util.py."""
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


def _make(D, l_max, order=2, seed=0, **kw):
    """(module on the GPU, oracle parameters) with the same weights; kw go to HyenaOperator (filter options)."""
    import hyena_dna_b200 as H
    g = torch.Generator().manual_seed(seed)
    P = O.init_params(D, l_max, order=order, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    P["in_proj.bias"] = 0.02 * torch.randn(P["in_proj.bias"].shape, generator=g)
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = H.HyenaOperator(D, l_max, order=order, emb_dim=5, w=10.0, **kw)
    op.load_state_dict(sd)
    if not kw.get("bias", True):
        P["filter_fn.bias"] = torch.zeros_like(P["filter_fn.bias"])      # use_bias=False: the filter bias is not applied
    return op.to(_dev()), P


def _truth(u, P, normalized=False):
    y32 = O.hyena_operator(u, P, normalized=normalized)
    y64 = O.hyena_operator(u.double(), O.to_dtype(P, torch.float64), normalized=normalized)
    return y32, y64


def _fft_min():
    import hyena_dna_b200 as H
    return H.ops.EXTEND_FFT_MIN_N


def _run(m, u, schedule, cache=None):
    """Feed u (on the GPU) to m (operator or backbone) by the schedule [(how, n), ...]; -> (outputs (B, L, D), cache)."""
    B, L, _ = u.shape
    cache = cache if cache is not None else m.allocate_decode_cache(B, L)
    outs, t = [], cache.t
    with torch.no_grad():
        for how, n in schedule:
            if how == "step":
                outs += [m.step(u[:, s:s + 1], cache) for s in range(t, t + n)]
            else:
                outs.append(getattr(m, how)(u[:, t:t + n], cache))
            t += n
    assert cache.t == t
    return torch.cat(outs, dim=1), cache


def _schedules():
    T = _fft_min()
    return {
        # extends start at every t mod 4 (t = 1, 3, 6, 12, 13, 76, 140)
        "mod4": (2, 64, [("prefill", 1), ("extend", 2), ("extend", 3), ("extend", 5), ("step", 1), ("extend", 1),
                         ("extend", 63), ("extend", 64), ("extend", 65)]),
        # chunks across the 1024-position partial boundaries, and both sides of the direct/FFT threshold
        "straddle": (1, 256, [("prefill", 1000), ("extend", 63), ("extend", 1000), ("step", 3), ("extend", 1500),
                              ("extend", T - 1), ("extend", T), ("extend", 2)]),
        "B3": (3, 32, [("prefill", 500), ("extend", 5), ("step", 2), ("extend", 65), ("extend", T - 1), ("extend", T)]),
        "B9": (9, 32, [("prefill", 100), ("extend", 3), ("extend", 1000), ("extend", 64), ("step", 1), ("extend", 1)]),
        "steps_first": (2, 64, [("step", 3), ("extend", 2), ("extend", 1500), ("extend", 63)]),
    }


@pytest.mark.parametrize("case", ["mod4", "straddle", "B3", "B9", "steps_first"])
def test_chunk_schedules_match_full_sequence(case):
    B, D, sched = _schedules()[case]
    L = sum(n for _, n in sched)
    op, P = _make(D, L)
    u = O.nucleotide_activations(B, L, D)[0]
    y, _ = _run(op, u.to(_dev()), sched)
    y32, y64 = _truth(u, P)
    t = 0
    for how, n in sched:                       # per chunk, so a failure names the chunk
        PU.check(y[:, t:t + n], y32[:, t:t + n], f"extend {case} {how} [{t}, {t + n})", ref64=y64[:, t:t + n])
        t += n


@pytest.mark.parametrize("variant", ["order3", "normalized", "trainable_deltas", "no_bias", "order4"])
def test_chunk_schedule_filter_variants(variant):
    B, D = 2, 32
    sched = [("prefill", 300), ("extend", 5), ("step", 1), ("extend", 64), ("extend", 7), ("extend", _fft_min())]
    L = sum(n for _, n in sched)
    kw, order, normalized = {}, 2, False
    if variant == "order3":
        order = 3
    elif variant == "order4":
        order = 4
    elif variant == "normalized":
        kw, normalized = {"normalized": True}, True
    elif variant == "trainable_deltas":
        kw = {"modulation_lr": 1e-3}
    elif variant == "no_bias":
        kw = {"bias": False}
    op, P = _make(D, L, order=order, **kw)
    u = O.nucleotide_activations(B, L, D)[0]
    y, _ = _run(op, u.to(_dev()), sched)
    y32, y64 = _truth(u, P, normalized=normalized)
    PU.check(y[:, 300:], y32[:, 300:], f"extend {variant}", ref64=y64[:, 300:])


@pytest.mark.parametrize("order", [2, 3])
def test_extend_on_fresh_cache_is_prefill(order):
    op, _ = _make(64, 2048, order=order)
    u = O.nucleotide_activations(2, 1500, 64)[0].to(_dev())
    with torch.no_grad():
        y_fwd = op(u)
        c1, c2 = op.allocate_decode_cache(2, 2048), op.allocate_decode_cache(2, 2048)
        y_ext = op.extend(u, c1)
        y_pre = op.prefill(u, c2)
    assert torch.equal(y_ext, y_fwd) and torch.equal(y_ext, y_pre)
    assert torch.equal(c1.h, c2.h) and torch.equal(c1.tail, c2.tail) and c1.t == c2.t == 1500


@pytest.mark.parametrize("side", [-1, 0])
def test_direct_and_fft_routes_agree_with_truth(side):
    """Both routes, each called through its own ops function, at the same (t, n) on either side of the threshold."""
    import hyena_dna_b200 as H
    dev = _dev()
    B, D, t = 2, 64, 3001
    n = _fft_min() + side
    assert H.ops.decode_extend_uses_fft(t, n) == (side == 0)
    op, P = _make(D, t + n)
    u = O.nucleotide_activations(B, t + n, D)[0]
    ud = u.to(dev)
    y32, y64 = _truth(u, P)
    for core in (H.ops.decode_extend_direct, H.ops.decode_extend_fft):
        cache = op.allocate_decode_cache(B, t + n)
        with torch.no_grad():
            op.prefill(ud[:, :t], cache)
            y = op._extend(ud[:, t:], cache, core)
        assert cache.t == t + n
        PU.check(y, y32[:, t:], f"extend {core.__name__} t={t} n={n}", ref64=y64[:, t:])


def _direct(u, sd, pos, dt, dev):
    """Outputs at positions ``pos`` of a long sequence by direct dot products over the history, in dtype dt on the GPU."""
    P = {k: v.to(dev, dt) for k, v in sd.items()}
    B, L, D = u.shape
    p = F.linear(u.to(dev, dt), P["in_proj.weight"], P["in_proj.bias"]).transpose(1, 2)
    uc = O.short_filter(p, P["short_filter.weight"], P["short_filter.bias"], L)
    del p
    x0, x1, v = uc.split(D, dim=1)
    g = (v * x1).contiguous()
    k = O.hyena_filter(L, P)[0].transpose(0, 1)                              # (D, L)
    rows = []
    for t in pos:
        c = (g[:, :, :t + 1] * k[:, :t + 1].flip(-1)).sum(-1) + P["filter_fn.bias"] * g[:, :, t]
        rows.append(c * x0[:, :, t])
    y_pre = torch.stack(rows, dim=1)                                          # (B, len(pos), D)
    return F.linear(y_pre, P["out_proj.weight"], P["out_proj.bias"]).cpu()


def test_chunked_prefill_at_full_length():
    """2^20 positions at D = 256 in four chunks against one forward, then the next 8 positions (one direct extend at
    t = 2^20 - 8) against direct fp64 dot products."""
    dev = _dev()
    L, D, N = 1 << 20, 256, 8
    op, P = _make(D, L)
    u = O.nucleotide_activations(1, L, D)[0]
    ud = u.to(dev)
    q = (L - N) // 4
    sched = [("prefill", q), ("extend", q), ("extend", q), ("extend", L - N - 3 * q), ("extend", N)]
    y, cache = _run(op, ud, sched)
    assert cache.t == L
    del cache
    with torch.no_grad():
        y_fwd = op(ud[:, :L - N]).cpu()
        P64 = {k: v.to(dev, torch.float64) for k, v in P.items()}
        y64 = O.hyena_operator(ud[:, :L - N].double(), P64).cpu()          # the oracle's fp64 truth, on the GPU
        del P64
    torch.cuda.empty_cache()
    PU.check(y[:, :L - N], y_fwd, "chunked prefill at L = 2^20 - 8 vs forward", ref64=y64)
    del y_fwd, y64
    pos = list(range(L - N, L))
    with torch.no_grad():
        y64 = _direct(u, P, pos, torch.float64, dev)
        y32 = _direct(u, P, pos, torch.float32, dev)
    PU.check(y[:, L - N:], y32, "extend of 8 at t = 2^20 - 8", ref64=y64)


@pytest.mark.parametrize("order", [2, 3])
def test_cache_state_matches_steps(order):
    """The same positions fed by one extend or by steps leave the same cache (h and tail within the bar, t exactly), and a
    later step continues alike from either."""
    dev = _dev()
    B, D, P0, n = 2, 64, 700, 400
    op, _ = _make(D, P0 + n + 1, order=order)
    u = O.nucleotide_activations(B, P0 + n + 1, D)[0].to(dev)
    _, ca = _run(op, u, [("prefill", P0), ("extend", n)], op.allocate_decode_cache(B, P0 + n + 1))
    _, cb = _run(op, u, [("prefill", P0), ("step", n)], op.allocate_decode_cache(B, P0 + n + 1))
    assert ca.t == cb.t == P0 + n
    for name in ("h", "tail"):
        a, b = getattr(ca, name), getattr(cb, name)
        PU.check(a, b, f"cache.{name} extend vs steps (order {order})")
    with torch.no_grad():
        ya, yb = op.step(u[:, -1:], ca), op.step(u[:, -1:], cb)
    PU.check(ya, yb, f"step after extend vs after steps (order {order})")


def _golden_backbone(case, mlp_cls):
    import hyena_dna_b200 as H
    z = np.load(os.path.join(GOLD, case + ".npz"))
    B, L, D, with_mlp = (int(v) for v in z["meta"])
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(mlp_cls, hidden_features=2 * D) if with_mlp else None
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return m.to(_dev()), z, L


@pytest.mark.parametrize("case", ["block_L128_D32_mlp", "block_L96_D16_nomlp"])
def test_backbone_extend_matches_reference_golden(case):
    import hyena_dna_b200 as H
    m, z, L = _golden_backbone(case, partial(H.Mlp, activation=partial(F.gelu, approximate="tanh")))
    x = torch.from_numpy(z["x"]).to(_dev())
    a, b = L // 3, L // 2
    sched = [("prefill", a), ("extend", b - a), ("step", 5), ("extend", L - b - 5)]
    y, cache = _run(m, x, sched)
    assert cache.t == L
    PU.check(y, torch.from_numpy(z["y"]), f"{case} extend y", ref64=torch.from_numpy(z["y64"]))


def test_inference_params_drive_extend():
    """Layers called the way the reference LMBackbone calls them (mixer_kwargs={"inference_params": cache}) with several
    positions after a prefill extend exactly as Backbone.extend does."""
    import hyena_dna_b200 as H
    dev = _dev()
    D, L = 32, 400
    m = H.Backbone(D, 3, partial(H.HyenaOperator, l_max=L, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=64)).to(dev)
    x = torch.randn(2, L, D, generator=torch.Generator().manual_seed(3)).to(dev)

    def via_kwargs(xs, cache):
        h, r = xs, None
        for layer in m.layers:
            h, r = layer(h, r, mixer_kwargs={"inference_params": cache})
        return H.Block._add_norm(h, r, m.ln_f)[0]

    cuts = [0, 100, 101, 164, 230, 400]
    c1, c2 = m.allocate_decode_cache(2, L), m.allocate_decode_cache(2, L)
    with torch.no_grad():
        # one position is a step either way; several positions after the prefill are an extend
        a = [m.prefill(x[:, :100], c1)] + [(m.step if e - s == 1 else m.extend)(x[:, s:e], c1)
                                           for s, e in zip(cuts[1:], cuts[2:])]
        b = [via_kwargs(x[:, s:e], c2) for s, e in zip(cuts, cuts[1:])]
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    assert c1.t == c2.t == L


def test_extend_is_deterministic():
    op, _ = _make(64, 3000)
    u = O.nucleotide_activations(3, 2900, 64)[0].to(_dev())
    sched = [("prefill", 1000), ("extend", 65), ("extend", 7), ("extend", _fft_min()), ("extend", 300)]
    assert torch.equal(_run(op, u, sched)[0], _run(op, u, sched)[0])


def test_extend_launches_and_profile():
    import hyena_dna_b200 as H
    dev = _dev()
    op, _ = _make(64, 4096, order=3)
    u = O.nucleotide_activations(1, 3001, 64)[0].to(dev)
    cache = op.allocate_decode_cache(1, 4096)
    with torch.no_grad():
        op.prefill(u[:, :2000], cache)
        H._lib.profile_begin()
        op.extend(u[:, 2000:2010], cache)            # direct route: hist, then (dot, combine) per recurrence
        prof = H._lib.profile_end()
        assert prof["decode_extend_hist"][1] == 1
        assert prof["decode_extend_dot"][1] == 2 and prof["decode_extend_combine"][1] == 2
        assert not {"decode_step", "decode_hist"} & set(prof)
        n0 = H.launch_count()
        op.extend(u[:, 2010:2020], cache)
        n_direct = H.launch_count() - n0
        assert n_direct == sum(v[1] for v in prof.values())
        H._lib.profile_begin()
        op.extend(u[:, 2020:2020 + _fft_min()], cache)       # FFT route: no direct kernel
        prof = H._lib.profile_end()
        assert "decode_extend_dot" not in prof
        assert prof["decode_extend_hist"][1] == 1 and prof["decode_extend_combine"][1] == 2
    assert cache.t == 2020 + _fft_min()
