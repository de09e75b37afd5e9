"""Full-size parity of the BASELINE.json configs against the reference's own GPU path.

The oracle (oracle/hyena_oracle.py: plain torch.fft / F.linear / F.conv1d, the reference's path restated and pinned
by tests/golden) runs on the SAME GPU in fp32 with TF32 off -- that IS the reference's PyTorch/cuFFT fftconv path
(src/models/sequence/hyena.py:59-88) -- and again in fp64 as the truth.  Tolerance policy: tests/parity_util.py.
All 15 parameter gradients are checked at every size.
"""
import gc

import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


# bytes of device memory the autograd oracle needs per (position, channel) in fp64 (saved spectra and activations of
# the whole operator); above the device's memory the fp64 truth runs on the host instead (same algorithm, fp64 either way)
_ORACLE64_BYTES_PER_ELEM = 320


def _truth_device(dev, B, L, D):
    free, _ = torch.cuda.mem_get_info(dev)
    return dev if B * L * D * _ORACLE64_BYTES_PER_ELEM < free else torch.device("cpu")


def _oracle_on(dev, dtype, u, P, dy):
    Pd = {k: v.to(device=dev, dtype=dtype) for k, v in P.items()}
    y, du, g = O.operator_fwd_bwd(u.to(device=dev, dtype=dtype), Pd, dy.to(device=dev, dtype=dtype))
    out = (y.cpu(), du.cpu(), {k: v.cpu() for k, v in g.items()})
    del Pd, y, du, g
    _free()
    return out


def _ours(dev, u, P, dy, D, L):
    import hyena_dna_b200 as H
    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = H.HyenaOperator(D, L, order=2, filter_order=64, emb_dim=5, w=10.0, lr_pos_emb=0.0)
    op.load_state_dict(sd, strict=True)
    op = op.to(dev)
    ug = u.to(dev).requires_grad_(True)
    y = op(ug)
    y.backward(dy.to(dev))
    torch.cuda.synchronize()
    out = (y.detach().cpu(), ug.grad.cpu(), {n: p.grad.cpu() for n, p in op.named_parameters() if p.grad is not None})
    del op, ug, y
    _free()
    return out


@pytest.mark.parametrize("name,B,L,D", [("small-32k", 8, 32768, 256), ("medium-160k", 4, 160000, 256),
                                        ("large-1m", 1, 1 << 20, 256)])
def test_baseline_config_full_width_against_reference_gpu_path(name, B, L, D):
    dev = _dev()
    g = torch.Generator().manual_seed(42)
    P = O.init_params(D, L, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    u, _ = O.nucleotide_activations(B, L, D, seed=2222)
    dy = torch.randn(B, L, D, generator=torch.Generator().manual_seed(1))
    y, du, grads = _ours(dev, u, P, dy, D, L)
    y32, du32, g32 = _oracle_on(dev, torch.float32, u, P, dy)
    y64, du64, g64 = _oracle_on(_truth_device(dev, B, L, D), torch.float64, u, P, dy)
    PU.check(y, y32, f"{name} y", ref64=y64)
    PU.check(du, du32, f"{name} du", ref64=du64)
    assert set(g32.keys()) <= set(grads.keys())
    assert len(g32) == 15
    for n in sorted(g32):
        PU.check(grads[n], g32[n], f"{name} grad {n}", ref64=g64[n], param_grad=True)


def test_large_1m_stress_inputs_full_width():
    """SURVEY.md S8(d) stress variant at the headline shape: u ~ N(0,1) i.i.d. instead of nucleotide embeddings."""
    dev = _dev()
    B, L, D = 1, 1 << 20, 256
    g = torch.Generator().manual_seed(7)
    P = O.init_params(D, L, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    u = torch.randn(B, L, D, generator=torch.Generator().manual_seed(0))
    dy = torch.randn(B, L, D, generator=torch.Generator().manual_seed(1))
    y, du, grads = _ours(dev, u, P, dy, D, L)
    y32, du32, g32 = _oracle_on(dev, torch.float32, u, P, dy)
    y64, du64, g64 = _oracle_on(_truth_device(dev, B, L, D), torch.float64, u, P, dy)
    PU.check(y, y32, "large-1m stress y", ref64=y64)
    PU.check(du, du32, "large-1m stress du", ref64=du64)
    for n in sorted(g32):
        PU.check(grads[n], g32[n], f"large-1m stress grad {n}", ref64=g64[n], param_grad=True)
