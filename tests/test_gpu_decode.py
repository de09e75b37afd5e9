"""Incremental decoding (HyenaOperator / Block / Backbone prefill + step, csrc/decode.cuh) against the fp64 truth of the
oracle on the whole sequence.  Tolerance policy: tests/parity_util.py."""
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
    # the model's initialisation (as smoke() and the operator parity tests use), with a non-zero in_proj bias so that the
    # bias the decoding kernels add is exercised
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


def _decode(op, u, P0, max_seqlen=None):
    """prefill u[:, :P0] (if P0 > 0), then step every later position; -> (B, L, D) outputs."""
    dev = _dev()
    B, L, D = u.shape
    cache = op.allocate_decode_cache(B, max_seqlen or L)
    ud = u.to(dev)
    outs = []
    with torch.no_grad():
        if P0 > 0:
            outs.append(op.prefill(ud[:, :P0], cache))
        for t in range(P0, L):
            outs.append(op.step(ud[:, t:t + 1], cache))
    assert cache.t == L
    return torch.cat(outs, dim=1)


@pytest.mark.parametrize("B,D,P0,N", [(2, 64, 0, 40), (2, 64, 1, 40), (2, 64, 1000, 40), (1, 256, 4090, 64)])
def test_continuation_matches_full_sequence(B, D, P0, N):
    L = P0 + N
    op, P = _make(D, L)
    u = O.nucleotide_activations(B, L, D)[0]
    y = _decode(op, u, P0)
    y32, y64 = _truth(u, P)
    if P0 > 0:
        PU.check(y[:, :P0], y32[:, :P0], f"decode prefill B{B} D{D} P{P0}", ref64=y64[:, :P0])
    PU.check(y[:, P0:], y32[:, P0:], f"decode steps B{B} D{D} P{P0} N{N}", ref64=y64[:, P0:])


@pytest.mark.parametrize("variant", ["order3", "normalized", "trainable_deltas", "no_bias", "order4"])
def test_continuation_filter_variants(variant):
    B, D, P0, N = 2, 32, 300, 24
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
    u = O.nucleotide_activations(B, P0 + N, D)[0]
    y = _decode(op, u, P0)
    y32, y64 = _truth(u, P, normalized=normalized)
    PU.check(y, y32, f"decode {variant}", ref64=y64)


def test_cached_filter_is_the_prefix_of_longer_filters():
    """k[j] does not depend on the length it is generated for: the cache's filter (Lcap taps) restricted to n taps is
    filter_channel_major(n), with normalized=True, trainable deltas and the class-default trainable z."""
    op, _ = _make(64, 3000, normalized=True, modulation_lr=1e-3, lr_pos_emb=1e-5)
    assert isinstance(op.filter_fn.pos_emb.z, torch.nn.Parameter)
    assert isinstance(op.filter_fn.modulation.deltas, torch.nn.Parameter)
    cache = op.allocate_decode_cache(1, 3000)
    F_, ld = 64, cache.h.shape[-1]
    k = cache.k[:F_ * ld].view(F_, ld)[:, ld - 3000:].flip(-1)
    with torch.no_grad():
        for n in (1, 7, 1024, 2999, 3000):
            torch.testing.assert_close(k[:, :n], op.filter_fn.filter_channel_major(n), rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("mode", ["tc", "lt"])
@pytest.mark.parametrize("order", [2, 3])
def test_prefill_is_forward(mode, order):
    import hyena_dna_b200 as H
    saved = H.ops._proj_mode
    H.ops._proj_mode = mode if mode == "tc" else ("lt" if H.ops.gemm_mode() == "bf16x9" else "torch")
    try:
        op, _ = _make(64, 2048, order=order)
        u = O.nucleotide_activations(2, 1500, 64)[0].to(_dev())
        with torch.no_grad():
            y_fwd = op(u)
            cache = op.allocate_decode_cache(2, 2048)
            y_pre = op.prefill(u, cache)
        assert torch.equal(y_fwd, y_pre)
        assert cache.t == 1500
    finally:
        H.ops._proj_mode = saved


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


def test_full_length_steps():
    dev = _dev()
    L, D, N = 1 << 20, 256, 8
    op, P = _make(D, L)
    u = O.nucleotide_activations(1, L, D)[0]
    y = _decode(op, u, L - N)[:, L - N:]
    pos = list(range(L - N, L))
    with torch.no_grad():
        y64 = _direct(u, P, pos, torch.float64, dev)
        y32 = _direct(u, P, pos, torch.float32, dev)
    PU.check(y, y32, "decode steps at L = 2^20", ref64=y64)


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
def test_backbone_decoding_matches_reference_golden(case):
    import hyena_dna_b200 as H
    m, z, L = _golden_backbone(case, partial(H.Mlp, activation=partial(F.gelu, approximate="tanh")))
    x = torch.from_numpy(z["x"]).to(_dev())
    half = L // 2
    cache = m.allocate_decode_cache(x.shape[0], L)
    with torch.no_grad():
        ys = [m.prefill(x[:, :half], cache)] + [m.step(x[:, t:t + 1], cache) for t in range(half, L)]
        y_fwd = m(x[:, :half])
    y = torch.cat(ys, dim=1)
    assert torch.equal(ys[0], y_fwd)                          # the backbone's prefill is its forward
    PU.check(y, torch.from_numpy(z["y"]), f"{case} decode y", ref64=torch.from_numpy(z["y64"]))


def test_mlp_runs_one_position():
    """Mlp (fc1 / fc2 on the wgmma GEMMs) on (B, 1, D), the shape a decoding step feeds it."""
    import hyena_dna_b200 as H
    dev = _dev()
    m = H.Mlp(64, hidden_features=256, activation=partial(F.gelu, approximate="tanh")).to(dev)
    x = torch.randn(3, 1, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        y = m(x)
        xd = x.double()
        y64 = F.linear(F.gelu(F.linear(xd, m.fc1.weight.double(), m.fc1.bias.double()), approximate="tanh"),
                       m.fc2.weight.double(), m.fc2.bias.double())
        y32 = F.linear(F.gelu(F.linear(x, m.fc1.weight, m.fc1.bias), approximate="tanh"), m.fc2.weight, m.fc2.bias)
    PU.check(y, y32, "Mlp L=1", ref64=y64)


def test_inference_params_drive_decoding():
    """Layers called the way the reference LMBackbone calls them (mixer_kwargs={"inference_params": cache}) decode exactly as
    prefill / step do; any other inference_params object leaves forward unchanged."""
    import hyena_dna_b200 as H
    dev = _dev()
    D, L, P0 = 32, 160, 100
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
        op = m.layers[0].mixer
        assert torch.equal(op(x), op(x, inference_params=object()))
    assert c1.t == c2.t == L


def test_decoding_is_deterministic():
    op, _ = _make(64, 3000)
    u = O.nucleotide_activations(2, 2100, 64)[0]
    assert torch.equal(_decode(op, u, 2000), _decode(op, u, 2000))


def test_step_launches_and_profile():
    import hyena_dna_b200 as H
    dev = _dev()
    op, _ = _make(64, 4096)
    u = O.nucleotide_activations(1, 3001, 64)[0].to(dev)
    cache = op.allocate_decode_cache(1, 4096)
    with torch.no_grad():
        n0 = H.launch_count()
        op.step(u[:, :1], cache)                          # t = 0: no history, the combine kernel only
        assert H.launch_count() - n0 == 1
        op.step(u[:, 1:2], cache)
        n0 = H.launch_count()
        op.step(u[:, 2:3], cache)
        assert H.launch_count() - n0 <= 2
        H._lib.profile_begin()
        op.step(u[:, 3:4], cache)
        prof = H._lib.profile_end()
    assert set(prof) == {"decode_step"} and prof["decode_step"][1] == 2
