"""CPU checks of the fftconv variants (k_rev, bidirectional): the oracle's restatement against the golden vectors generated
from the unmodified reference fftconv_ref (tests/golden/make_golden_fftconv.py), and the time-domain decomposition the
sm_90a host side uses (hyena_dna_b200/fftconv.py: RevCorrFunc, fftconv_ref) against that restatement."""
import os

import numpy as np
import pytest
import torch

from oracle import hyena_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fftconv_variants.npz")
NAMES = ["krev_L100", "krev_L257", "bidir_L128", "bidir_L101"]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_fftconv_variants_match_reference_golden(name):
    z = np.load(GOLD)
    T = lambda k: torch.from_numpy(z[f"{name}/{k}"])
    B, H, L, with_rev, bidir = (int(v) for v in z[f"{name}/cfg"])
    for dt, tag, tol in ((torch.float32, "", 2e-6), (torch.float64, "64", 1e-12)):
        u, k, D = (T(x).to(dt).requires_grad_(True) for x in ("u", "k", "D"))
        kr = T("krev").to(dt).requires_grad_(True) if with_rev else None
        y = O.fftconv_ref(u, k, D, k_rev=kr, bidirectional=bool(bidir))
        y.backward(T("dy").to(dt))
        s = float(T("y" + tag).abs().max())
        assert float((y.detach() - T("y" + tag)).abs().max()) <= tol * max(1.0, s)
        for got, want in ((u.grad, "du"), (k.grad, "dk"), (D.grad, "dD")) + (((kr.grad, "dkrev"),) if with_rev else ()):
            w = T(want + tag)
            assert float((got - w).abs().max()) <= 10 * tol * max(1.0, float(w.abs().max())), want


@pytest.mark.parametrize("L,with_rev,bidir", [(64, True, False), (37, True, False), (64, False, True), (37, False, True),
                                              (2, False, True), (1, False, True)])
def test_time_domain_decomposition_equals_the_reference_formula(L, with_rev, bidir):
    g = torch.Generator().manual_seed(L + 7 * with_rev + 13 * bidir)
    u = torch.randn(2, 3, L, generator=g, dtype=torch.float64)
    k = torch.randn(3, L, generator=g, dtype=torch.float64)
    kr = torch.randn(3, L, generator=g, dtype=torch.float64) if with_rev else None
    D = torch.randn(3, generator=g, dtype=torch.float64)
    ref = O.fftconv_ref(u, k, D, k_rev=kr, bidirectional=bidir)
    dec = O.fftconv_variants_time_domain(u, k, D, k_rev=kr, bidirectional=bidir)
    torch.testing.assert_close(dec, ref, rtol=1e-10, atol=1e-10)


def test_rev_corr_backward_formulas():
    """Backward of y = corr(u, k_rev) as hyena_dna_b200.fftconv.RevCorrFunc computes it: du = causal conv(dy, k_rev),
    dk_rev[m] = sum_t u[t] dy[t - m] -- against autograd of the reference formula."""
    L = 48
    g = torch.Generator().manual_seed(3)
    u = torch.randn(2, 3, L, generator=g, dtype=torch.float64, requires_grad=True)
    kr = torch.randn(3, L, generator=g, dtype=torch.float64, requires_grad=True)
    k0 = torch.zeros(3, L, dtype=torch.float64); D0 = torch.zeros(3, dtype=torch.float64)
    dy = torch.randn(2, 3, L, generator=g, dtype=torch.float64)
    O.fftconv_ref(u, k0, D0, k_rev=kr).backward(dy)
    du = O.fftconv_direct(dy, kr.detach(), D0)                       # causal conv(dy, k_rev)
    dk = torch.zeros(3, L, dtype=torch.float64)
    for m in range(L):
        dk[:, m] = (u.detach()[..., m:] * dy[..., : L - m]).sum((0, 2))
    torch.testing.assert_close(du, u.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dk, kr.grad, rtol=1e-10, atol=1e-10)
