"""Windowed decoding steps (ops.decode_window_refresh / decode_win_step, csrc/decode.cuh decode_win_step_kernel), reached
through HyenaOperator / Backbone step, against the fp64 truth of the oracle.  The window constants are lowered so that
windows open at small sizes, except in the full-length test.  Tolerance policy: tests/parity_util.py."""
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


def _ops():
    import hyena_dna_b200 as H
    return H.ops


@pytest.fixture
def small_windows(monkeypatch):
    """Windows of W positions open after 2 steps at any history."""
    ops = _ops()

    def set_(W=64, min_t=0, after=2):
        monkeypatch.setattr(ops, "WINDOW", W)
        monkeypatch.setattr(ops, "WINDOW_MIN_T", min_t)
        monkeypatch.setattr(ops, "WINDOW_AFTER_STEPS", after)
    set_()
    return set_


def _make(D, l_max, order=2, seed=0, **kw):
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
        P["filter_fn.bias"] = torch.zeros_like(P["filter_fn.bias"])
    return op.to(_dev()), P


def _truth(u, P, normalized=False):
    y32 = O.hyena_operator(u, P, normalized=normalized)
    y64 = O.hyena_operator(u.double(), O.to_dtype(P, torch.float64), normalized=normalized)
    return y32, y64


def _run(m, u, schedule, cache=None):
    """Feed u (on the GPU) to m by the schedule [(how, n), ...], how in prefill / extend / step / fft (an extend forced onto
    the FFT route) -> (outputs (B, L, D), cache)."""
    import hyena_dna_b200 as H
    B, L, _ = u.shape
    cache = cache if cache is not None else m.allocate_decode_cache(B, L)
    outs, t = [], cache.t
    with torch.no_grad():
        for how, n in schedule:
            if how == "step":
                outs += [m.step(u[:, s:s + 1], cache) for s in range(t, t + n)]
            elif how == "fft":
                outs.append(m._extend(u[:, t:t + n], cache.for_module(m), H.ops.decode_extend_fft))
            else:
                outs.append(getattr(m, how)(u[:, t:t + n], cache))
            t += n
    assert cache.t == t
    return torch.cat(outs, dim=1), cache


def _check_schedule(op, P, B, D, sched, what, normalized=False):
    L = sum(n for _, n in sched)
    u = O.nucleotide_activations(B, L, D)[0]
    y, cache = _run(op, u.to(_dev()), sched)
    y32, y64 = _truth(u, P, normalized=normalized)
    t = 0
    for how, n in sched:
        PU.check(y[:, t:t + n], y32[:, t:t + n], f"{what} {how} [{t}, {t + n})", ref64=y64[:, t:t + n])
        t += n
    return cache


@pytest.mark.parametrize("B,P0", [(1, 1021), (3, 998), (9, 1)])
def test_steps_across_windows(small_windows, B, P0):
    """Prefill, then steps over more than three windows of 64: every t mod 4, window bases on both sides of a 1024-position
    chunk boundary (P0 = 1021, 998) and from the start of the sequence (P0 = 1)."""
    D, N = 32, 3 * 64 + 41
    op, P = _make(D, P0 + N)
    cache = _check_schedule(op, P, B, D, [("prefill", P0), ("step", N)], f"window steps B{B} P{P0}")
    assert cache.win_wc > 0 and cache.win_b > P0 + 2 * 64
    assert cache.window_nbytes == 4 * B * D * 64


@pytest.mark.parametrize("variant", ["order3", "order4", "normalized", "trainable_deltas", "no_bias"])
def test_window_filter_variants(small_windows, variant):
    small_windows(W=32)
    B, D, P0, N = 2, 32, 300, 100
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
    op, P = _make(D, P0 + N, order=order, **kw)
    cache = _check_schedule(op, P, B, D, [("prefill", P0), ("step", N)], f"window {variant}", normalized)
    assert cache.win_wc > 0 and tuple(cache.win_f.shape) == (order - 1, B, D, 32)


@pytest.mark.parametrize("case", ["direct_inside", "fft_inside", "across_end", "to_lcap"])
def test_extend_interleaved_with_windows(small_windows, case):
    """Window [b, b + 64) opened at t = 503 + 2 = 505 -> b = 504.  An extend inside it (direct or FFT route) keeps it for
    the following steps; one across its end closes it; generation runs up to Lcap, where the last window is clipped."""
    B, D = 2, 32
    scheds = {
        "direct_inside": [("prefill", 503), ("step", 5), ("extend", 7), ("step", 30), ("extend", 3), ("step", 90)],
        "fft_inside": [("prefill", 503), ("step", 5), ("fft", 9), ("step", 20), ("fft", 30), ("step", 70)],
        "across_end": [("prefill", 503), ("step", 40), ("extend", 50), ("step", 1), ("step", 80), ("extend", 64),
                       ("step", 3)],
        "to_lcap": [("prefill", 503), ("step", 150)],
    }
    sched = scheds[case]
    L = sum(n for _, n in sched)
    op, P = _make(D, L)
    _check_schedule(op, P, B, D, sched, f"interleaved {case}")


def test_launches_and_profile(small_windows):
    import hyena_dna_b200 as H
    ops = H.ops
    dev = _dev()
    op, _ = _make(64, 4096, order=3)
    u = O.nucleotide_activations(1, 3000, 64)[0].to(dev)
    # below the thresholds: the parent's launches and bits
    small_windows(W=64, min_t=10 ** 9, after=2)
    ca, cb = op.allocate_decode_cache(1, 4096), op.allocate_decode_cache(1, 4096)
    with torch.no_grad():
        op.prefill(u[:, :2001], ca)
        op.prefill(u[:, :2001], cb)
        H._lib.profile_begin()
        ya = [op.step(u[:, t:t + 1], ca) for t in range(2001, 2011)]
        prof = H._lib.profile_end()
        assert set(prof) == {"decode_step"} and prof["decode_step"][1] == 10 * 2 * 2
        p_list = []
        for t in range(2001, 2011):                           # the plain route called directly
            p_t = F.linear(u[:, t], op.in_proj.weight).contiguous()
            ib, sw, sb = op._decode_params()
            p_list.append(F.linear(ops.decode_step(p_t, ib, sw, sb, cb), op.out_proj.weight, op.out_proj.bias))
            cb.t += 1
        assert all(torch.equal(a.reshape(-1), b.reshape(-1)) for a, b in zip(ya, p_list))
        assert ca.win_wc == 0 and ca.win_f is None
        # thresholds lowered: the count is already past 2, so the next step refreshes (b = 2008)
        small_windows(W=64, min_t=0, after=2)
        H._lib.profile_begin()
        op.step(u[:, 2011:2012], ca)
        prof = H._lib.profile_end()
        assert (ca.win_b, ca.win_wc) == (2008, 64)
        assert prof["decode_win_step"][1] == 2 * 2 and "decode_step" not in prof
        assert len(prof) > 1                                  # the refresh's FFT kernels
        H._lib.profile_begin()
        for t in range(2012, 2072):                           # in the window up to its last position 2071
            op.step(u[:, t:t + 1], ca)
        prof = H._lib.profile_end()
        assert set(prof) == {"decode_win_step"} and prof["decode_win_step"][1] == 60 * 2 * 2
        H._lib.profile_begin()
        op.step(u[:, 2072:2073], ca)                          # expired: refresh, then t = b: one launch per recurrence
        prof = H._lib.profile_end()
        assert ca.win_b == 2072 and prof["decode_win_step"][1] == 2
        n0 = H.launch_count()
        op.step(u[:, 2073:2074], ca)
        assert H.launch_count() - n0 == 4


@pytest.mark.parametrize("order", [2, 3])
def test_cache_state_after_windowed_steps(small_windows, order):
    """The same steps with and without windows leave h and tail within the bar; a later step and a later extend continue
    alike from either."""
    dev = _dev()
    B, D, P0, n = 2, 64, 700, 200
    op, _ = _make(D, P0 + n + 40, order=order)
    u = O.nucleotide_activations(B, P0 + n + 40, D)[0].to(dev)
    _, ca = _run(op, u[:, :P0 + n], [("prefill", P0), ("step", n)], op.allocate_decode_cache(B, P0 + n + 40))
    small_windows(min_t=10 ** 9)
    _, cb = _run(op, u[:, :P0 + n], [("prefill", P0), ("step", n)], op.allocate_decode_cache(B, P0 + n + 40))
    assert ca.win_wc > 0 and cb.win_wc == 0
    for name in ("h", "tail"):
        PU.check(getattr(ca, name), getattr(cb, name), f"cache.{name} windowed vs plain steps (order {order})")
    small_windows()
    ya, _ = _run(op, u, [("step", 1), ("extend", 39)], ca)
    yb, _ = _run(op, u, [("step", 1), ("extend", 39)], cb)
    PU.check(ya, yb, f"step + extend after windowed vs plain steps (order {order})")


def test_windowed_steps_are_deterministic(small_windows):
    op, _ = _make(64, 3000)
    u = O.nucleotide_activations(3, 2300, 64)[0].to(_dev())
    sched = [("prefill", 2001), ("step", 150), ("extend", 5), ("step", 144)]
    assert torch.equal(_run(op, u, sched)[0], _run(op, u, sched)[0])


def _golden_backbone(case):
    import hyena_dna_b200 as H
    z = np.load(os.path.join(GOLD, case + ".npz"))
    B, L, D, with_mlp = (int(v) for v in z["meta"])
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=2 * D, activation=partial(F.gelu, approximate="tanh")) if with_mlp else None
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return m.to(_dev()), z, L


@pytest.mark.parametrize("case", ["block_L128_D32_mlp", "block_L96_D16_nomlp"])
def test_backbone_golden_through_windows(small_windows, case):
    small_windows(W=16)
    m, z, L = _golden_backbone(case)
    x = torch.from_numpy(z["x"]).to(_dev())
    y, cache = _run(m, x, [("prefill", 9), ("step", L - 9)])
    assert all(c.win_wc > 0 for c in cache.layers)
    PU.check(y, torch.from_numpy(z["y"]), f"{case} windowed decode y", ref64=torch.from_numpy(z["y64"]))


def test_inference_params_through_windows(small_windows):
    import hyena_dna_b200 as H
    small_windows(W=16)
    dev = _dev()
    D, L, P0 = 32, 200, 50
    m = H.Backbone(D, 3, partial(H.HyenaOperator, l_max=L, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=64)).to(dev)
    x = torch.randn(2, L, D, generator=torch.Generator().manual_seed(3)).to(dev)

    def via_kwargs(xs, cache):
        h, r = xs, None
        for layer in m.layers:
            h, r = layer(h, r, mixer_kwargs={"inference_params": cache})
        return H.Block._add_norm(h, r, m.ln_f)[0]

    c1, c2 = m.allocate_decode_cache(2, L), m.allocate_decode_cache(2, L)
    with torch.no_grad():
        a = [m.prefill(x[:, :P0], c1)] + [m.step(x[:, t:t + 1], c1) for t in range(P0, L)]
        b = [via_kwargs(x[:, :P0], c2)] + [via_kwargs(x[:, t:t + 1], c2) for t in range(P0, L)]
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    assert all(c.win_wc > 0 for c in c1.layers) and c1.t == c2.t == L


def _direct(u, sd, pos, dt, dev):
    """Outputs at positions ``pos`` by direct dot products over the whole history, in dtype dt on the GPU."""
    P = {k: v.to(dev, dt) for k, v in sd.items()}
    B, L, D = u.shape
    p = F.linear(u.to(dev, dt), P["in_proj.weight"], P["in_proj.bias"]).transpose(1, 2)
    uc = O.short_filter(p, P["short_filter.weight"], P["short_filter.bias"], L)
    del p
    x0, x1, v = uc.split(D, dim=1)
    g = (v * x1).contiguous()
    k = O.hyena_filter(L, P)[0].transpose(0, 1)
    rows = []
    for t in pos:
        c = (g[:, :, :t + 1] * k[:, :t + 1].flip(-1)).sum(-1) + P["filter_fn.bias"] * g[:, :, t]
        rows.append(c * x0[:, :, t])
    y_pre = torch.stack(rows, dim=1)
    return F.linear(y_pre, P["out_proj.weight"], P["out_proj.bias"]).cpu()


def test_full_length_generation_with_shipped_windows():
    """D = 256, l_max = 2^20, the shipped constants: prefill 2^20 - N, then steps to the cache end over at least two full
    windows and a clipped last one.  Sampled positions (every window edge +-2 and a random sample) against fp64 dot
    products over the whole history."""
    import hyena_dna_b200 as H
    ops = H.ops
    dev = _dev()
    L, D, W, S = 1 << 20, 256, ops.WINDOW, ops.WINDOW_AFTER_STEPS
    N = S + 2 * W + W // 2 + 3
    assert L - N >= ops.WINDOW_MIN_T
    op, P = _make(D, L)
    u = O.nucleotide_activations(1, L, D)[0]
    ud = u.to(dev)
    cache = op.allocate_decode_cache(1, L)
    ys, bases = [], []
    with torch.no_grad():
        op.prefill(ud[:, :L - N], cache)
        for t in range(L - N, L):
            ys.append(op.step(ud[:, t:t + 1], cache))
            if cache.win_wc and (not bases or bases[-1] != cache.win_b):
                bases.append(cache.win_b)
    assert cache.t == L and len(bases) >= 3
    y = torch.cat(ys, dim=1).cpu()
    del cache, ys
    torch.cuda.empty_cache()
    edges = {p for b in bases for e in (b, min(b + W, L)) for p in range(e - 2, e + 3)}
    rng = np.random.default_rng(0)
    pos = sorted({p for p in edges if L - N <= p < L} | set(rng.integers(L - N, L, 24).tolist()))
    with torch.no_grad():
        y64 = _direct(u, P, pos, torch.float64, dev)
        y32 = _direct(u, P, pos, torch.float32, dev)
    PU.check(y[:, [p - (L - N) for p in pos]], y32, "windowed steps at L = 2^20", ref64=y64)
