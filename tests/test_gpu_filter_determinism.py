"""The implicit filter's backward is bitwise reproducible at the benchmark's shape.

Stage 2 (the sequence-length reductions that turn the stage-1 arrays into the parameter gradients) sums per-CTA partials
in a fixed order, so two runs on the same inputs return the same bits.  It used to flush its accumulators with atomic
adds, whose order changed from run to run.
"""
import pytest
import torch

from tests.test_gpu_filter_paths import _H, _dev, case, case_inputs, expected_grads, make_filter

gpu = pytest.mark.gpu


@gpu
def test_filter_backward_is_bitwise_reproducible():
    """D = 256, L = 2^20, E = 5 (bench.py's operator): k and every filter gradient of two fwd+bwd runs are equal."""
    H = _H()
    dev = _dev()
    c = case(256, 1 << 20, init_std=0.02, modulation_lr=1e-3, seed=7)
    P, dk = case_inputs(c)
    dk = dk.to(dev)
    runs = []
    for _ in range(2):
        f = make_filter(H, P, c, dev)
        k = f.filter_channel_major(c["L"])
        k.backward(dk)
        params = dict(f.named_parameters())
        runs.append({"k": k.detach().clone(), **{n: params[n].grad.clone() for n in expected_grads(c)}})
        del f, k
    torch.cuda.synchronize()
    for n, a in runs[0].items():
        b = runs[1][n]
        assert torch.equal(a, b), f"{n}: two runs differ in {(a != b).sum().item()} of {a.numel()} elements"
