"""Host planning of decode.StepGraph with the capture and the replay stubbed (no GPU needed): which graph runs, when the
window refresh runs, how the host position, the step count and the device position move, the argument and state errors,
and the C ABI of the device-position steps with its guards."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch

_lib = import_module("hyena_dna_b200._lib")

P = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


NAMES = ("hyena_b200_decode_step_dev", "hyena_b200_decode_win_step_dev", "hyena_b200_decode_branch_step_dev",
         "hyena_b200_decode_pos_advance")


def test_dev_step_abi_present():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header


def _step(pos=P, o=0, order=2, v_in=None, p_t=P, t_max=64, Lcap=64, B=1, cache_B=1, h=P):
    return _lib.lib().hyena_b200_decode_step_dev(p_t, P, P, P, P, P, h, P, P, v_in, P, P, pos, B, cache_B, 8, order, o,
                                                 t_max, Lcap, None)


def test_dev_step_abi_guards():
    assert _step(pos=None) != 0 and "device position" in _err()
    assert _step(pos=ctypes.c_void_p(258)) != 0 and "device position" in _err()
    assert _step(t_max=0) != 0 and "position bound" in _err()
    assert _step(t_max=65) != 0 and "position bound" in _err()
    assert _step(o=1) != 0 and "recurrence" in _err()
    assert _step(p_t=None) != 0 and "recurrence 0 needs" in _err()
    assert _step(o=1, order=3) != 0 and "v_in" in _err()
    assert _step(B=2) != 0 and "differs from the decode cache" in _err()
    assert _step(h=ctypes.c_void_p(260)) != 0 and "aligned" in _err()
    L = _lib.lib()
    assert L.hyena_b200_decode_win_step_dev(P, P, P, P, P, P, P, P, P, None, P, P, P, P, 1, 1, 8, 2, 0, 0, 64, None) != 0
    assert "window width" in _err()
    assert L.hyena_b200_decode_win_step_dev(P, P, P, P, P, P, P, P, P, None, P, P, P, P, 1, 1, 8, 2, 0, 65, 64, None) != 0
    assert "window width" in _err()
    assert L.hyena_b200_decode_win_step_dev(P, P, P, P, P, P, P, P, P, None, P, P, None, P, 1, 1, 8, 2, 0, 8, 64, None) != 0
    assert "null pointer" in _err()
    for H in (6, 0, 68):
        assert L.hyena_b200_decode_branch_step_dev(P, P, P, P, P, P, P, P, P, None, P, P, P, P, P, 2, 8, 2, 0, H, 64,
                                                   None) != 0
        assert "branch history width" in _err()
    assert L.hyena_b200_decode_branch_step_dev(P, P, P, P, P, P, P, P, P, None, P, P, P, None, P, 2, 8, 2, 0, 8, 64,
                                               None) != 0 and "null pointer" in _err()
    assert L.hyena_b200_decode_pos_advance(None, None) != 0 and "device position" in _err()


# ---------------------------------------------------------------------------------------------- host planning (stubbed)
def _H():
    import hyena_dna_b200 as H
    return H


def _cpu_cache(op, B=1, lcap=None):
    H = _H()
    lcap = lcap or op.l_max
    ld = (lcap + 3) // 4 * 4
    D, O = op.d_model, op.order
    F, C = (O - 1) * D, (O + 1) * D
    return H.DecodeCache(op, B, lcap, lcap, torch.zeros(F * ld + 4), torch.zeros(F), torch.zeros(O - 1, B, D, ld),
                         torch.zeros(B, C, 2), torch.zeros(B, C), torch.zeros(B, D, (lcap + 1023) // 1024))


class _FakeGraph:
    """Records the route and the device position of every replay, then advances it as the graph's last kernel does."""

    def __init__(self, sg, route, log):
        self.sg, self.route, self.log = sg, route, log

    def replay(self):
        pos = self.sg.cache.pos
        self.log.append((self.route, tuple(pos.tolist())))
        pos[0] += 1


@pytest.fixture
def stubbed(monkeypatch):
    """Small window constants, capture and refresh stubbed: -> the log of captures, refreshes and replays."""
    H = _H()
    ops = H.ops
    monkeypatch.setattr(ops, "WINDOW_MIN_T", 8)
    monkeypatch.setattr(ops, "WINDOW_AFTER_STEPS", 3)
    monkeypatch.setattr(ops, "WINDOW", 8)
    log = []

    def capture(self, route):
        log.append(("capture", route))
        if route == "window":
            for c in self.caches:
                if c.win_f is None:
                    c.win_f = torch.zeros(c.order - 1, c.batch_size, c.d_model, ops.WINDOW)
        self.cache.sync_position()
        return _FakeGraph(self, route, log), ("out", route)

    def refresh(c):
        c.win_b, c.win_wc = ops.decode_window_bounds(c.t, c.lcap)
        log.append(("refresh", c.t))
    monkeypatch.setattr(H.StepGraph, "_capture", capture)
    monkeypatch.setattr(ops, "decode_window_refresh", refresh)
    return log


def test_routes_refreshes_and_positions(stubbed):
    """Plain graph below WINDOW_MIN_T; the first step at WINDOW_MIN_T refreshes and switches to the window graph (no
    WINDOW_AFTER_STEPS run of plain steps); refresh at each window end; a window clipped at Lcap; the host position and
    step count advance per replay and the device position is the host's at every replay."""
    H = _H()
    op = H.HyenaOperator(8, 30, emb_dim=5)
    c = _cpu_cache(op)
    c.t = 5
    g = H.StepGraph(op, c)
    assert stubbed == [("capture", "plain")] and g.plan() == ("plain", False)
    u = torch.zeros(1, 1, 8)
    outs = [g.step(u) for _ in range(25)]
    assert c.t == 30 and c.steps == 25
    assert outs[:3] == [("out", "plain")] * 3 and set(outs[3:]) == {("out", "window")}
    events = [e for e in stubbed if e[0] in ("capture", "refresh")]
    assert events == [("capture", "plain"), ("refresh", 8), ("capture", "window"), ("refresh", 16), ("refresh", 24)]
    replays = [e for e in stubbed if e[0] in ("plain", "window")]
    assert [p[0] for _, p in replays] == list(range(5, 30))
    assert all(p[1] == (p[0] - p[0] % 8 if p[0] >= 8 else 0) for _, p in replays)
    assert (c.win_b, c.win_wc) == (24, 6)                         # clipped at Lcap = 30
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        g.step(u)
    assert c.t == 30 and len(stubbed) == len(events) + len(replays)


def test_eager_steps_in_between_resync(stubbed):
    """Positions moved by eager work between replays (here by hand) reach the device before the next replay."""
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op)
    c.t = 2
    g = H.StepGraph(op, c)
    u = torch.zeros(1, 1, 8)
    g.step(u)
    c.t += 3                                       # e.g. an extend of 3
    c.steps = 0
    g.step(u)
    assert stubbed[-1] == ("plain", (6, 0, 0)) and c.t == 7 and c.steps == 1
    assert tuple(c.pos.tolist()) == (7, 0, 0) and c._pos_state.value == (7, 0, 0)


def test_stack_shares_one_position(stubbed):
    """A Backbone's graph advances every layer's host position once per token and all layers read one device position."""
    H = _H()
    m = H.Backbone(8, 3, partial(H.HyenaOperator, l_max=64, emb_dim=5))
    cache = H.DecodeCache.stack(_cpu_cache(layer.mixer, B=2) for layer in m.layers)
    for c in cache.layers:
        c.t = 10
    g = H.StepGraph(m, cache, 2)
    for _ in range(3):
        g.step(torch.zeros(2, 1, 8))
    assert [c.t for c in cache.layers] == [13] * 3 and [c.steps for c in cache.layers] == [3] * 3
    assert all(c.pos is cache.pos for c in cache.layers)
    assert stubbed[:4] == [("capture", "window")] + [("refresh", 10)] * 3            # every layer's window, once
    assert [p for r, p in stubbed if r == "window"] == [(10, 8, 0), (11, 8, 0), (12, 8, 0)]
    cache.layers[1].t += 1
    with pytest.raises(H.HyenaB200Error, match="disagree"):
        cache.sync_position()


def test_branched_route_and_horizon(stubbed):
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op, B=3)
    c._branched, c.base, c.hc, c.t = True, 20, 8, 22
    c.f, c.parent = torch.zeros(1, 1, 8, 8), torch.zeros(3, dtype=torch.int32)
    g = H.StepGraph(op, c, 3)
    u = torch.zeros(3, 1, 8)
    for _ in range(6):
        g.step(u)
    assert c.t == 28 and c.steps == 0
    assert [e for e in stubbed if e[0] == "branch"][-1] == ("branch", (27, 0, 20))
    with pytest.raises(H.HyenaB200Error, match="horizon"):
        g.step(u)
    with pytest.raises(H.HyenaB200Error, match="horizon"):
        H.StepGraph(op, c, 3)
    assert c.t == 28


def test_argument_and_state_errors(stubbed):
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    c = _cpu_cache(op, B=2)
    c.t = 4
    with pytest.raises(H.HyenaB200Error, match="batch size"):
        H.StepGraph(op, c, 3)
    with pytest.raises(H.HyenaB200Error, match="DecodeCache"):
        H.StepGraph(op, object())
    with pytest.raises(H.HyenaB200Error, match="HyenaOperator, Block or Backbone"):
        H.StepGraph(torch.nn.Linear(2, 2), c)
    with pytest.raises(H.HyenaB200Error, match="residual"):
        H.StepGraph(op, c, residual=True)
    with pytest.raises(H.HyenaB200Error, match="not allocated for this"):
        H.StepGraph(H.HyenaOperator(8, 64, emb_dim=5), c)
    g = H.StepGraph(op, c)
    n = len(stubbed)
    for bad in (torch.zeros(1, 1, 8), torch.zeros(2, 2, 8), torch.zeros(2, 1, 8, dtype=torch.float64)):
        with pytest.raises(H.HyenaB200Error, match="differs from the captured"):
            g.step(bad)
    with pytest.raises(H.HyenaB200Error, match="captured without a residual"):
        g.step(torch.zeros(2, 1, 8), torch.zeros(2, 1, 8))
    for name in ("h", "tail"):
        old = getattr(c, name)
        setattr(c, name, old.clone())
        with pytest.raises(H.HyenaB200Error, match="replaced"):
            g.step(torch.zeros(2, 1, 8))
        setattr(c, name, old)
    assert len(stubbed) == n and c.t == 4
    g.step(torch.zeros(2, 1, 8))
    assert c.t == 5
