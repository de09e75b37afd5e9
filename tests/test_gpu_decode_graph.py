"""Decode steps captured in CUDA graphs (decode.StepGraph, the device-position kernels of csrc/decode.cuh) against eager
``step`` on an identical cache: every output and the cache state after the run must be the same bits."""
from functools import partial

import pytest
import torch

from oracle import hyena_oracle as O

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _op(D, l_max, order=2, seed=0):
    torch.manual_seed(seed)
    op = _H().HyenaOperator(D, l_max, order=order, emb_dim=5, w=10.0)
    with torch.no_grad():
        op.in_proj.bias.normal_(0, 0.02)
    return op.to(_dev())


def _backbone(D, l_max, n_layer=3, seed=0):
    H = _H()
    torch.manual_seed(seed)
    m = H.Backbone(D, n_layer, partial(H.HyenaOperator, l_max=l_max, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True)
    return m.to(_dev())


def _twins(m, B, lcap, u, P):
    """Two caches of m filled by the same prefill of u[:, :P]: identical bits."""
    caches = [m.allocate_decode_cache(B, lcap) for _ in range(2)]
    with torch.no_grad():
        for c in caches:
            m.prefill(u[:, :P], c)
    a, b = (c.layers or [c] for c in caches)
    for x, y in zip(a, b):
        assert torch.equal(x.h, y.h) and torch.equal(x.tail, y.tail)
    return caches


def _same_state(ca, cb):
    for a, b in zip(ca.layers or [ca], cb.layers or [cb]):
        assert a.t == b.t and a.steps == b.steps and (a.win_b, a.win_wc) == (b.win_b, b.win_wc)
        assert torch.equal(a.h, b.h) and torch.equal(a.tail, b.tail)
        if a.win_wc:
            assert torch.equal(a.win_f[..., :a.win_wc], b.win_f[..., :b.win_wc])


def _run_both(m, ce, cg, u, t0, n):
    """n steps from position t0: eager on ce, StepGraph on cg; every output compared bit for bit."""
    H = _H()
    g = H.StepGraph(m, cg, u.shape[0], u.dtype)
    n0 = H.launch_count()
    with torch.no_grad():
        for i in range(t0, t0 + n):
            ye = m.step(u[:, i:i + 1], ce)
            yg = g.step(u[:, i:i + 1])
            assert torch.equal(ye, yg), f"position {i}: max diff {(ye - yg).abs().max().item():.3e}"
    return g, H.launch_count() - n0


@pytest.mark.parametrize("order", [2, 3])
def test_operator_plain_route(order):
    """64 graph steps from a short prefill, no library call in a replay, then eager step and extend on the graph's cache
    match an all-eager run."""
    H = _H()
    dev = _dev()
    B, D, P, n, lcap = 2, 64, 300, 64, 1024
    op = _op(D, lcap, order)
    u = O.nucleotide_activations(B, lcap, D)[0].to(dev)
    ce, cg = _twins(op, B, lcap, u, P)
    g, eager_launches = _run_both(op, ce, cg, u, P, n)
    # the eager steps launched 2 (O-1) kernels each, the replays none
    assert eager_launches == 2 * (order - 1) * n
    _same_state(ce, cg)
    with torch.no_grad():
        s = P + n
        assert torch.equal(op.step(u[:, s:s + 1], ce), op.step(u[:, s:s + 1], cg))
        assert torch.equal(op.extend(u[:, s + 1:s + 6], ce), op.extend(u[:, s + 1:s + 6], cg))
        # and the graph goes on from there (its device position is re-synced)
        s += 6
        assert torch.equal(op.step(u[:, s:s + 1], ce), g.step(u[:, s:s + 1]))
    _same_state(ce, cg)


def test_operator_crosses_window_min_t():
    """From below WINDOW_MIN_T across it and two window ends (refreshes between replays) into a window clipped at Lcap."""
    H = _H()
    ops = H.ops
    dev = _dev()
    W, T = ops.WINDOW, ops.WINDOW_MIN_T
    lcap = T + 2 * W + 1000
    B, D, P = 1, 16, T - 40
    end = T + 2 * W + 100
    op = _op(D, lcap)
    u = O.nucleotide_activations(B, lcap, D)[0].to(dev)
    ce, cg = _twins(op, B, lcap, u, P)
    g, _ = _run_both(op, ce, cg, u, P, end - P)
    assert set(g._graphs) == {"plain", "window"}
    assert cg.win_b == T + 2 * W and cg.win_wc == lcap - cg.win_b
    _same_state(ce, cg)


def test_backbone_mlp_crosses_window_min_t():
    H = _H()
    ops = H.ops
    dev = _dev()
    W, T = ops.WINDOW, ops.WINDOW_MIN_T
    lcap = T + 2 * W + 1000
    B, D, P = 2, 16, T - 24
    end = T + 2 * W + 20
    m = _backbone(D, lcap)
    u = torch.randn(B, lcap, D, generator=torch.Generator().manual_seed(1)).to(dev)
    ce, cg = _twins(m, B, lcap, u, P)
    g, _ = _run_both(m, ce, cg, u, P, end - P)
    assert set(g._graphs) == {"plain", "window"}
    _same_state(ce, cg)
    with torch.no_grad():
        assert torch.equal(m.extend(u[:, end:end + 3], ce), m.extend(u[:, end:end + 3], cg))


def test_block_with_and_without_residual():
    H = _H()
    dev = _dev()
    B, D, P, lcap = 2, 32, 100, 512
    m = _backbone(D, lcap, n_layer=2)
    u = torch.randn(B, lcap, D, generator=torch.Generator().manual_seed(2)).to(dev)
    ce, cg = _twins(m, B, lcap, u, P)
    b0, b1 = m.layers
    g0, g1 = b0.capture_step(cg), b1.capture_step(cg, residual=True)
    with torch.no_grad():
        for i in range(P, P + 20):
            he, re = b0.step(u[:, i:i + 1], None, ce)
            he, re = b1.step(he, re, ce)
            hg, rg = g0.step(u[:, i:i + 1])
            hg, rg = g1.step(hg, rg)
            assert torch.equal(he, hg) and torch.equal(re, rg)
    _same_state(ce, cg)


def test_branches_then_select():
    """8 branches of 2 parent rows stepped by graphs; select on both; a fresh graph on the selection, up to the horizon;
    one more step raises before any launch."""
    H = _H()
    dev = _dev()
    B, D, P, horizon, lcap = 2, 32, 1001, 64, 2048
    op = _op(D, lcap, order=3)
    u = O.nucleotide_activations(B, P, D)[0].to(dev)
    ub = O.nucleotide_activations(8, horizon, D, seed=5)[0].to(dev)
    pe, pg = _twins(op, B, lcap, u, P)
    rows = [0, 1, 1, 0, 0, 1, 0, 1]
    be, bg = pe.fork(rows, horizon), pg.fork(rows, horizon)
    b = P - P % 4
    _run_both(op, be, bg, torch.cat([torch.zeros(8, P, D, device=dev), ub], 1), P, 20)
    _same_state(be, bg)
    idx = [3, 3, 0, 7, 1, 6, 2, 2]
    se, sg = be.select(idx), bg.select(idx)
    ub2 = torch.cat([torch.zeros(8, P + 20, D, device=dev), ub[:, 20:]], 1)
    g, _ = _run_both(op, se, sg, ub2, P + 20, b + horizon - P - 20)
    assert sg.t == b + horizon
    _same_state(se, sg)
    n0, h0 = H.launch_count(), sg.h.clone()
    with pytest.raises(H.HyenaB200Error, match="horizon"):
        g.step(ub[:, :1])
    assert H.launch_count() == n0 and sg.t == b + horizon and torch.equal(sg.h, h0)


def test_errors_before_any_work():
    H = _H()
    dev = _dev()
    B, D, lcap = 1, 32, 40
    op = _op(D, lcap)
    u = O.nucleotide_activations(B, lcap, D)[0].to(dev)
    c = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(u[:, :30], c)
    g = op.capture_step(c)
    n0 = H.launch_count()
    for bad in (u[:, :2, :], u[:, :1].double(), u[:, :1].cpu(), torch.cat([u[:, :1]] * 2)):
        with pytest.raises(H.HyenaB200Error, match="differs from the captured"):
            g.step(bad)
    assert H.launch_count() == n0 and c.t == 30
    with torch.no_grad():
        for i in range(30, 40):
            g.step(u[:, i:i + 1])
    n0 = H.launch_count()
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        g.step(u[:, :1])
    assert H.launch_count() == n0 and c.t == 40
    with pytest.raises(H.HyenaB200Error, match="past the cache"):
        op.capture_step(c)
    # a buffer the graph reads replaced behind its back
    c2 = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(u[:, :30], c2)
    g2 = op.capture_step(c2)
    c2.tail = c2.tail.clone()
    with pytest.raises(H.HyenaB200Error, match="replaced"):
        g2.step(u[:, 30:31])
    assert c2.t == 30


def test_replay_is_one_graph_launch():
    """torch.profiler: a replay issues no CUDA API call but the graph launch (and the input copy)."""
    dev = _dev()
    B, D, P, lcap = 1, 64, 200, 1024
    op = _op(D, lcap)
    u = O.nucleotide_activations(B, lcap, D)[0].to(dev)
    c = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(u[:, :P], c)
        g = op.capture_step(c)
        g.step(u[:, P:P + 1])
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            g.step(u[:, P + 1:P + 2])
            torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("cudaGraphLaunch" in n for n in names)
    launches = [n for n in names if n in ("cudaLaunchKernel", "cuLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernelEx")]
    assert launches == [], launches


def test_own_weight_images_survive_other_work_on_the_capture_stream(monkeypatch):
    """The Mlp GEMMs of a graph use weight-image scratch held by the StepGraph, not the library's per-stream entry: a
    second, wider graph captured on the same (pooled) stream, and eager GEMMs there, replace that entry and free its
    memory, and the first graph still replays bit-exact without writing into memory it does not own."""
    H = _H()
    ops = H.ops
    dev = _dev()
    B, D, P, lcap = 1, 32, 100, 512
    m = _backbone(D, lcap, n_layer=2)
    u = torch.randn(B, lcap, D, generator=torch.Generator().manual_seed(4)).to(dev)
    ce, cg = _twins(m, B, lcap, u, P)
    g = m.capture_step(cg)
    side = g._side
    assert g._scratch and all(s is not v for s in g._scratch for v in ops._wimg_cache.values())
    with torch.no_grad():
        for i in range(P, P + 4):
            assert torch.equal(m.step(u[:, i:i + 1], ce), g.step(u[:, i:i + 1]))
        # a wider backbone captured on the same stream, then eager GEMMs there with a still larger weight image
        monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: side)
        wide = _backbone(512, 256, n_layer=1)
        cw = wide.allocate_decode_cache(1, 256)
        wide.prefill(torch.randn(1, 8, 512, device=dev), cw)
        gw = wide.capture_step(cw)
        assert gw._side is side
        with torch.cuda.stream(side):
            x = torch.randn(1, 4, 1024, device=dev)
            ops.proj_gemm(x, 0, torch.randn(4096, 1024, device=dev), False, 0)
            fill = [torch.full((8 << 20,), 7, dtype=torch.uint8, device=dev) for _ in range(8)]
        torch.cuda.current_stream().wait_stream(side)
        for i in range(P + 4, P + 12):
            assert torch.equal(m.step(u[:, i:i + 1], ce), g.step(u[:, i:i + 1]))
            gw.step(torch.randn(1, 1, 512, device=dev))
        torch.cuda.synchronize()
    assert all(bool((f == 7).all()) for f in fill)
    _same_state(ce, cg)


def test_profiling_while_capturing():
    """With the library's per-launch timing on, a capture records no events into the graph and the position advance counts
    under no kind: only the warm-up steps' dot and combine kernels show as decode_step launches."""
    H = _H()
    dev = _dev()
    B, D, P, lcap = 1, 32, 100, 512
    op = _op(D, lcap)
    u = O.nucleotide_activations(B, lcap, D)[0].to(dev)
    c = op.allocate_decode_cache(B, lcap)
    with torch.no_grad():
        op.prefill(u[:, :P], c)
        H._lib.profile_begin()
        n0 = H.launch_count()
        g = op.capture_step(c)
        for i in range(P, P + 3):
            g.step(u[:, i:i + 1])
        prof = H._lib.profile_end()
    warm = H.StepGraph.WARMUP
    assert prof["decode_step"][1] == 2 * warm
    # the capture counts its launches once (3 per step), the replays none
    assert H.launch_count() - n0 == 3 * (warm + 1)
