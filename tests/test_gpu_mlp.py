"""Block MLP (hyena_dna_b200.Mlp: fc1 -> GELU -> fc2 on the wgmma projection kernels with the GELU fused in) against the
reference composition F.linear -> F.gelu -> F.linear in fp32 (TF32 off) and in fp64, against the reference golden
backbone, and for its memory and determinism properties.  Tolerance policy: tests/parity_util.py."""
import gc
import os
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import parity_util as PU

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _inputs(B, L, D, H, bias, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, D, generator=g)
    W1 = torch.randn(H, D, generator=g) / D ** 0.5
    W2 = torch.randn(D, H, generator=g) / H ** 0.5
    b1 = 0.5 * torch.randn(H, generator=g) if bias else None
    b2 = 0.1 * torch.randn(D, generator=g) if bias else None
    dy = torch.randn(B, L, D, generator=g)
    return x, W1, b1, W2, b2, dy


def _reference(dev, dtype, approximate, x, W1, b1, W2, b2, dy):
    """The reference Mlp.forward (flash_attn/modules/mlp.py:26-30) and its autograd, results on the host."""
    t = lambda v: None if v is None else v.to(dev, dtype).requires_grad_(True)
    xx, w1, bb1, w2, bb2 = t(x), t(W1), t(b1), t(W2), t(b2)
    y = F.linear(F.gelu(F.linear(xx, w1, bb1), approximate=approximate), w2, bb2)
    y.backward(dy.to(dev, dtype))
    g = lambda v: None if v is None else v.grad.cpu()
    out = (y.detach().cpu(), g(xx), g(w1), g(bb1), g(w2), g(bb2))
    del xx, w1, bb1, w2, bb2, y
    _free()
    return out


def _ours(dev, approximate, x, W1, b1, W2, b2, dy):
    import hyena_dna_b200 as H
    D, Hd = W1.shape[1], W1.shape[0]
    m = H.Mlp(D, hidden_features=Hd, activation=partial(F.gelu, approximate=approximate), bias1=b1 is not None,
              bias2=b2 is not None).to(dev)
    with torch.no_grad():
        m.fc1.weight.copy_(W1); m.fc2.weight.copy_(W2)
        if b1 is not None:
            m.fc1.bias.copy_(b1); m.fc2.bias.copy_(b2)
    xx = x.to(dev).requires_grad_(True)
    y = m(xx)
    y.backward(dy.to(dev))
    g = lambda p: None if p is None else p.grad.cpu()
    out = (y.detach().cpu(), xx.grad.cpu(), g(m.fc1.weight), g(m.fc1.bias), g(m.fc2.weight), g(m.fc2.bias))
    del m, xx, y
    _free()
    return out


_NAMES = ("y", "dx", "dW1", "db1", "dW2", "db2")


def _compare(tag, ours, r32, r64):
    for n, o, a, b in zip(_NAMES, ours, r32, r64):
        if a is None:
            assert o is None, f"{tag} {n}: unexpected gradient"
            continue
        PU.check(o, a, f"{tag} {n}", ref64=b, param_grad=n not in ("y", "dx"))


@pytest.mark.parametrize("approximate", ["tanh", "none"])
@pytest.mark.parametrize("B,L,D,Hd", [(2, 1000, 128, 512), (1, 4096, 256, 1024), (3, 777, 64, 256), (1, 513, 32, 64)])
def test_mlp_matches_torch_fp32_and_fp64(B, L, D, Hd, approximate):
    dev = _dev()
    args = _inputs(B, L, D, Hd, True, seed=B * 7 + L + D + Hd)
    ours = _ours(dev, approximate, *args)
    r32 = _reference(dev, torch.float32, approximate, *args)
    r64 = _reference(dev, torch.float64, approximate, *args)
    _compare(f"mlp {approximate} B{B} L{L} D{D} H{Hd}", ours, r32, r64)


@pytest.mark.parametrize("approximate", ["tanh", "none"])
def test_mlp_without_biases(approximate):
    dev = _dev()
    args = _inputs(2, 1000, 128, 512, False, seed=5)
    ours = _ours(dev, approximate, *args)
    assert ours[3] is None and ours[5] is None
    _compare(f"mlp no-bias {approximate}", ours, _reference(dev, torch.float32, approximate, *args),
             _reference(dev, torch.float64, approximate, *args))


def test_backbone_with_mlp_matches_reference_golden():
    """The golden backbone (tests/golden/make_golden_block.py, the UNMODIFIED reference Block + Mlp) with hyena_dna_b200.Mlp
    as mlp_cls: the reference state_dict loads strictly and y, dx and every parameter gradient match."""
    import hyena_dna_b200 as H
    dev = _dev()
    z = np.load(os.path.join(GOLD, "block_L128_D32_mlp.npz"))
    B, L, D, with_mlp = (int(v) for v in z["meta"])
    assert with_mlp
    mixer = partial(H.HyenaOperator, l_max=L, order=2, filter_order=64, emb_dim=5, w=10.0, shift=0.0, lr_pos_emb=0.0)
    mlp = partial(H.Mlp, hidden_features=2 * D, activation=partial(F.gelu, approximate="tanh"))
    m = H.Backbone(D, 2, mixer, mlp_cls=mlp, layer_norm_epsilon=1e-5, residual_in_fp32=True)
    assert all(isinstance(layer.mlp, H.Mlp) for layer in m.layers)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
    m.load_state_dict(sd, strict=True)
    m = m.to(dev)
    x = torch.from_numpy(z["x"]).to(dev).requires_grad_(True)
    y = m(x)
    y.backward(torch.from_numpy(z["dy"]).to(dev))
    PU.check(y, torch.from_numpy(z["y"]), "mlp golden y", ref64=torch.from_numpy(z["y64"]))
    PU.check(x.grad, torch.from_numpy(z["dx"]), "mlp golden dx", ref64=torch.from_numpy(z["dx64"]))
    got = {n: p.grad for n, p in m.named_parameters() if p.grad is not None}
    want = [k[5:] for k in z.files if k.startswith("grad/")]
    assert any(".mlp.fc1." in n for n in want) and set(want) <= set(got)
    for n in want:
        PU.check(got[n], torch.from_numpy(z["grad/" + n]), f"mlp golden grad {n}", ref64=torch.from_numpy(z["grad64/" + n]),
                 param_grad=True)


def test_mlp_full_size_against_torch_gpu_path():
    """B = 1, L = 2^20, D = 256, H = 1024 (the HyenaDNA d_inner = 4 d_model at the headline length)."""
    dev = _dev()
    args = _inputs(1, 1 << 20, 256, 1024, True, seed=11)
    ours = _ours(dev, "tanh", *args)
    r32 = _reference(dev, torch.float32, "tanh", *args)
    r64 = _reference(dev, torch.float64, "tanh", *args)
    _compare("mlp full-size", ours, r32, r64)


def test_mlp_is_deterministic_and_runs_the_library_kernels():
    import hyena_dna_b200 as H
    dev = _dev()
    assert H.ops.proj_mode() == "tc"
    m = H.Mlp(256, activation=partial(F.gelu, approximate="tanh")).to(dev)
    x = torch.randn(2, 3000, 256, device=dev, requires_grad=True)
    dy = torch.randn(2, 3000, 256, device=dev)
    outs = []
    for _ in range(2):
        x.grad = None
        m.zero_grad(set_to_none=True)
        n0 = H.launch_count()
        y = m(x)
        torch.cuda.synchronize()
        n1 = H.launch_count()
        y.backward(dy)
        torch.cuda.synchronize()
        n2 = H.launch_count()
        assert n1 - n0 == 4 and n2 - n1 == 8         # fwd: 2 x (prep + gemm); bwd: 2 x (prep + gemm) + 2 x (wgrad + reduce)
        outs.append([y.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    H._lib.profile_begin()
    m(x).backward(dy)
    prof = H._lib.profile_end()
    assert {"proj_gemm", "proj_gemm<gelu>", "proj_gemm<dgelu>", "proj_wgrad", "proj_wgrad<gelu>"} <= set(prof), prof


def test_mlp_saves_one_hidden_tensor():
    import hyena_dna_b200 as H
    dev = _dev()
    B, L, D, Hd = 2, 1024, 64, 256
    saved = []

    def pack(t):
        saved.append(tuple(t.shape))
        return t

    m = H.Mlp(D, hidden_features=Hd, activation=partial(F.gelu, approximate="tanh")).to(dev)
    x = torch.randn(B, L, D, device=dev, requires_grad=True)
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        y = m(x)
    hidden = [s for s in saved if int(np.prod(s)) == B * L * Hd]
    assert hidden == [(B, Hd, L)], saved
    assert sum(int(np.prod(s)) for s in saved) == B * L * D + B * L * Hd + 2 * D * Hd, saved   # x, a, W1, W2
    y.sum().backward()
    assert x.grad is not None and m.fc1.weight.grad is not None


def test_mlp_tf32_opt_in_runs_the_reference_composition():
    """torch.backends.cuda.matmul.allow_tf32 switches the projections to the library GEMM path (ops.proj_mode); the MLP
    then is the reference's own F.linear + F.gelu composition."""
    import hyena_dna_b200 as H
    dev = _dev()
    m = H.Mlp(64, activation=partial(F.gelu, approximate="tanh"), return_residual=True).to(dev)
    x = torch.randn(2, 100, 64, device=dev)
    try:
        torch.backends.cuda.matmul.allow_tf32 = True
        mode = H.ops.proj_mode()
        y, res = m(x)
        want = m.fc2(F.gelu(m.fc1(x), approximate="tanh"))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    assert res is x
    if mode != "tc":
        assert torch.equal(y, want)
