"""Unbounded decode caches (max_seqlen=None, DESIGN.md section 4.20) without a GPU: the slide plan over a table of cases
and exhaustively, the layout and allocation errors, the prompt-length errors before any device work, and the host
bookkeeping of a slide (dropped, window, every layer of a stack)."""
from functools import partial
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")
ops = import_module("hyena_dna_b200.ops")
decode = import_module("hyena_dna_b200.decode")


def _H():
    import hyena_dna_b200 as H
    return H


def _cpu_cache(op, B=2, t=0):
    """An unbounded cache with the layout's shapes on the CPU (allocate_decode_cache itself needs the GPU)."""
    H = _H()
    lcap = decode.unbounded_lcap(op.l_max)
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    c = H.DecodeCache(op, B, None, lcap, torch.zeros(F * ld + 4), torch.zeros(F), torch.zeros(O - 1, B, D, ld),
                      torch.zeros(B, C, 2), torch.zeros(B, C), torch.zeros(B, D, (lcap + 1023) // 1024), reach=op.l_max)
    c.t = t
    return c


# ---------------------------------------------------------------------------------------------- the layout
@pytest.mark.parametrize("l_max,S,lcap", [(61, 64, 128), (64, 64, 132), (1026, 1028, 2060), (4096, 4096, 8196),
                                          (4099, 4096, 8200), (1 << 17, 4096, (1 << 17) + 4100)])
def test_slide_room_and_lcap(l_max, S, lcap):
    assert decode.slide_room(l_max) == S and decode.unbounded_lcap(l_max) == lcap
    assert lcap % 4 == 0 and lcap >= l_max + S + 3


# ---------------------------------------------------------------------------------------------- the plan, by table
# (t, n, lk, win_b, win_wc) -> (shift, t', keep) or an error; lk = 61 (S = 64, Lcap = 128) and lk = 4099 (S = 4096,
# Lcap = 8200): neither a multiple of 4
PLAN = [
    # room left: no slide, whatever t
    ((0, 1, 61, 0, 0), (0, 0, False)), ((60, 1, 61, 0, 0), (0, 60, False)), ((61, 64, 61, 0, 0), (0, 61, False)),
    ((127, 1, 61, 0, 0), (0, 127, False)), ((64, 64, 61, 0, 0), (0, 64, False)), ((63, 65, 61, 0, 0), (0, 63, False)),
    ((124, 4, 61, 120, 8), (0, 124, True)),
    # at Lcap: m = t - lk + 1 rounded down to a multiple of 4
    ((128, 1, 61, 0, 0), (-68, 60, False)), ((128, 64, 61, 0, 0), (-68, 60, False)), ((128, 65, 61, 0, 0), (-68, 60, False)),
    ((125, 4, 61, 0, 0), (-64, 61, False)), ((127, 2, 61, 0, 0), (-64, 63, False)), ((126, 3, 61, 0, 0), (-64, 62, False)),
    # Lcap - n < t: the piece of S = 64 positions and of S + 1
    ((65, 64, 61, 0, 0), (-4, 61, False)), ((67, 64, 61, 0, 0), (-4, 63, False)), ((68, 64, 61, 0, 0), (-8, 60, False)),
    ((67, 65, 61, 0, 0), (-4, 63, False)), ((64, 65, 61, 0, 0), (-4, 60, False)),
    # too many positions even after the slide
    ((62, 67, 61, 0, 0), "even after a slide"), ((60, 69, 61, 0, 0), "even after a slide"),
    ((10, 200, 61, 0, 0), "even after a slide"),
    # a window that holds t is kept when m <= win_b, closed otherwise; one that does not hold t is closed
    ((128, 1, 61, 68, 60), (-68, 60, False)), ((127, 2, 61, 68, 60), (-64, 63, True)),
    ((127, 2, 61, 64, 64), (-64, 63, True)), ((127, 2, 61, 60, 68), (-64, 63, False)),
    ((127, 2, 61, 0, 128), (-64, 63, False)), ((127, 2, 61, 64, 60), (-64, 63, False)),
    # lk = 4099
    ((8200, 1, 4099, 0, 0), (-4100, 4100, False)), ((8199, 1, 4099, 0, 0), (0, 8199, False)),
    ((4105, 4096, 4099, 0, 0), (-4, 4101, False)), ((4106, 4097, 4099, 0, 0), (-8, 4098, False)),
    ((8195, 4096, 4099, 4100, 4096), (-4096, 4099, True)), ((8191, 10, 4099, 4092, 4100), (-4092, 4099, True)),
    ((4098, 4103, 4099, 0, 0), "even after a slide"),
]


@pytest.mark.parametrize("case,want", PLAN)
def test_slide_plan_table(case, want):
    t, n, lk, wb, wc = case
    lcap = decode.unbounded_lcap(lk)
    if isinstance(want, str):
        with pytest.raises(_lib.HyenaB200Error, match=want):
            ops.decode_slide_plan(t, n, lk, lcap, wb, wc)
    else:
        assert ops.decode_slide_plan(t, n, lk, lcap, wb, wc) == want


# (t, win_b, win_wc) of a step at lk = 2^16 (Lcap = 69636) -> (shift, t'): a step slides early rather than open a window
# shorter than WINDOW; a held window, a refresh of full width or t below WINDOW_MIN_T need no slide
STEP = [((69632, 0, 0), (-4096, 65536)), ((69632, 65536, 4096), (-4096, 65536)), ((65544, 0, 0), (-8, 65536)),
        ((65543, 0, 0), (0, 65543)), ((65540, 0, 0), (0, 65540)), ((69000, 65536, 4096), (0, 69000)),
        ((69635, 69632, 4), (0, 69635)), ((69636, 69632, 4), (-4100, 65536)), ((65536, 0, 0), (0, 65536))]


@pytest.mark.parametrize("case,want", STEP)
def test_slide_plan_step_keeps_windows_full(case, want):
    lk = 1 << 16
    lcap = decode.unbounded_lcap(lk)
    t, wb, wc = case
    shift, t2, _ = ops.decode_slide_plan(t, 1, lk, lcap, wb, wc, step=True)
    assert (shift, t2) == want
    assert ops.decode_slide_plan(t, 1, lk, lcap, wb, wc)[0] == (shift if t == lcap else 0)     # an extend does not
    if not (wc and wb <= t2 - shift < wb + wc):
        assert ops.decode_window_bounds(t2, lcap)[1] == ops.WINDOW


def test_slide_plan_step_exhaustive():
    """Every position a step can see at l_max 2^16 and 4099 + 2^16: the step slides exactly when t is at Lcap or a refresh
    would open a window shorter than WINDOW, and afterwards every refresh opens a full window."""
    for lk in (1 << 16, (1 << 16) + 4099):
        lcap = decode.unbounded_lcap(lk)
        for t in range(lk - 8, lcap + 1):
            shift, t2, _ = ops.decode_slide_plan(t, 1, lk, lcap, step=True)
            short = t >= ops.WINDOW_MIN_T and ops.decode_window_bounds(t, lcap)[1] < ops.WINDOW
            assert (shift != 0) == (t == lcap or short), (lk, t)
            if t2 >= ops.WINDOW_MIN_T:
                assert ops.decode_window_bounds(t2, lcap)[1] == ops.WINDOW, (lk, t)


def test_slide_plan_exhaustive():
    """Every reachable t and n <= S + 4: the plan drops no position an output at t or later reaches, shifts by a multiple
    of 4, leaves room for the n positions and never fails for n <= S; without need it does not slide."""
    for lk in list(range(1, 40)) + [255, 1026]:
        S, lcap = decode.slide_room(lk), decode.unbounded_lcap(lk)
        for t in range(0, lcap + 1):
            for n in list(range(1, 6)) + list(range(S - 4, S + 5)):
                if n < 1:
                    continue
                for wb, wc in ((0, 0), (t - t % 4, 4), (max(t - 40, 0) // 4 * 4, 64)):
                    try:
                        shift, t2, keep = ops.decode_slide_plan(t, n, lk, lcap, wb, wc)
                    except _lib.HyenaB200Error:
                        assert n > S, (lk, t, n)
                        continue
                    m = -shift
                    assert m % 4 == 0 and 0 <= m <= max(t - lk + 1, 0) and t2 == t - m and t2 + n <= lcap
                    assert (m == 0) == (t + n <= lcap)
                    holds = wc > 0 and wb <= t < wb + wc
                    assert keep == (holds and m <= wb)


# ---------------------------------------------------------------------------------------------- allocation and bytes
def test_layout_nbytes_counts_the_slack():
    H = _H()
    for B, D, O, l_max in [(1, 256, 2, 1 << 17), (2, 64, 3, 1026), (3, 8, 2, 61)]:
        lcap = decode.unbounded_lcap(l_max)
        ld, F, C = lcap, (O - 1) * D, (O + 1) * D
        want = 4 * (F * ld + 4 + F + (O - 1) * B * D * ld + 2 * B * C + B * C + B * D * -(-lcap // 1024))
        assert H.DecodeCache.layout_nbytes(B, D, O, lcap) == want
        assert want > H.DecodeCache.layout_nbytes(B, D, O, l_max)
        assert H.DecodeCache.layout_nbytes(B, D, O, lcap, torch.bfloat16) == want - 2 * (O - 1) * B * D * ld
    op = H.HyenaOperator(8, 61, emb_dim=5, order=3)
    c = _cpu_cache(op)
    assert c.nbytes == H.DecodeCache.layout_nbytes(2, 8, 3, 128)
    assert c.unbounded and c.slide == 64 and c.dropped == 0 and c.max_seqlen is None


def test_allocation_errors():
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    for kw, msg in [(dict(batch_size=0, max_seqlen=None), "batch_size 0"), (dict(batch_size=0, max_seqlen=5), "must be"),
                    (dict(batch_size=2, max_seqlen=None), "CUDA"), (dict(batch_size=2, max_seqlen=8), "CUDA")]:
        with pytest.raises(H.HyenaB200Error, match=msg):
            op.allocate_decode_cache(**kw)
    big = H.HyenaOperator(4, (1 << 20) - 4096, emb_dim=3)
    with pytest.raises(H.HyenaB200Error, match="more than the 1048576"):
        big.allocate_decode_cache(1, None)
    assert H.DecodeCache.check_allocation(1, None, (1 << 20) - 4100) == (1 << 20) - 4100
    bb = H.Backbone(8, 2, partial(H.HyenaOperator, l_max=64, emb_dim=5))
    bb.layers[1].mixer.l_max = 128
    with pytest.raises(H.HyenaB200Error, match="same l_max"):
        bb.allocate_decode_cache(1, None)
    with pytest.raises(H.HyenaB200Error, match="same l_max"):
        H.DecodeCache.stack([_cpu_cache(H.HyenaOperator(8, 64, emb_dim=5)), _cpu_cache(H.HyenaOperator(8, 61, emb_dim=5))])


# ---------------------------------------------------------------------------------------------- errors before device work
@pytest.fixture
def no_device(monkeypatch):
    """Every device entry point fails the test if reached."""
    H = _H()
    for name in ("core_forward", "decode_hist", "decode_admit", "decode_admit_packed", "decode_shift", "proj_gemm",
                 "add_layer_norm", "filter_spectrum", "decode_step_auto", "decode_extend"):
        monkeypatch.setattr(H.ops, name, lambda *a, _n=name, **k: pytest.fail(f"device work ({_n}) before validation"))
    return H


@pytest.mark.parametrize("order", [2, 3])
def test_prompts_longer_than_l_max_raise_before_device_work(no_device, order):
    H = no_device
    mixer = partial(H.HyenaOperator, l_max=61, emb_dim=5, order=order)
    op, bb = mixer(8), H.Backbone(8, 2, mixer)
    n0 = H.launch_count()
    u = torch.zeros(2, 62, 8)
    first = [lambda: op.prefill(u, _cpu_cache(op), lengths=[62, 3]),
             lambda: op.extend(u, _cpu_cache(op), lengths=[62, 3])]
    if order == 2:
        cu = torch.tensor([0, 62, 70])
        first += [lambda: op.prefill(torch.zeros(70, 8), _cpu_cache(op), cu_seqlens=cu),
                  lambda: op.admit(torch.zeros(70, 8), _cpu_cache(op, t=100), [0, 1], cu_seqlens=cu)]
    for call in first:
        with pytest.raises(H.HyenaB200Error, match="exceeds l_max = 61.*extend"):      # forward's input checks, with the hint
            call()
    calls = [lambda: op.prefill(u, _cpu_cache(op)),
             lambda: op.admit(u, _cpu_cache(op, t=100), [0, 1]),
             lambda: bb.prefill(u, H.DecodeCache.stack([_cpu_cache(layer.mixer) for layer in bb.layers])),
             lambda: bb.admit(u, H.DecodeCache.stack([_cpu_cache(layer.mixer, t=90) for layer in bb.layers]), [0, 1])]
    for call in calls:
        with pytest.raises(H.HyenaB200Error, match="exceeds l_max = 61.*extend"):
            call()
    # l_max positions are accepted: the checks pass on to the device check
    with pytest.raises(H.HyenaB200Error, match="CUDA"):
        op.prefill(torch.zeros(2, 61, 8), _cpu_cache(op))
    assert H.launch_count() == n0


# ---------------------------------------------------------------------------------------------- bookkeeping of a slide
def test_slide_bookkeeping(no_device, monkeypatch):
    H = no_device
    shifts = []

    def shift(cache, s):
        shifts.append((id(cache), s))
        start = cache.start if cache.start is not None else (0,) * cache.batch_size
        cache.set_start([max(x + s, 0) for x in start])
        cache.t += s
        cache.win_b = max(cache.win_b + s, 0)
    monkeypatch.setattr(H.ops, "decode_shift", shift)
    op = H.HyenaOperator(8, 61, emb_dim=5)
    c = _cpu_cache(op, t=100)
    assert c._make_room(28) == 0 and not shifts                       # 100 + 28 = Lcap: no slide
    c.win_b, c.win_wc = 100, 28
    assert c._make_room(29) == 40 and shifts == [(id(c), -40)] and (c.t, c.dropped) == (60, 40)
    assert (c.win_b, c.win_wc) == (60, 28)                            # 40 <= win_b: the window is kept
    c.t, c.win_b, c.win_wc = 128, 20, 120
    assert c._make_room(1) == 68 and (c.t, c.dropped, c.win_wc) == (60, 108, 0)     # 68 > win_b: closed
    c.reset_window()
    assert c.dropped == 0
    # a stack slides every layer by the same shift; a bounded cache never slides
    stack = H.DecodeCache.stack([_cpu_cache(op, t=128), _cpu_cache(op, t=128)])
    shifts.clear()
    assert stack.unbounded and stack.slide == 64 and stack._make_room(1) == 68
    assert [s for _, s in shifts] == [-68, -68] and stack.dropped == 68 and stack.t == 60
    assert {layer.t for layer in stack.layers} == {60}
    bounded = H.DecodeCache(op, 2, 61, 61, torch.zeros(64 + 4), torch.zeros(8), torch.zeros(1, 2, 8, 64),
                            torch.zeros(2, 24, 2), torch.zeros(2, 24), torch.zeros(2, 8, 1))
    bounded.t = 61
    assert not bounded.unbounded and bounded.slide is None and bounded._make_room(1) == 0 and bounded.dropped == 0
    # a branch of an unbounded cache is not unbounded
    br = _cpu_cache(op, t=10)
    br.reach = None
    assert not br.unbounded
