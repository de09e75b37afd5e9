"""The projection GEMM's schedule (csrc/proj_gemm.cuh): every CTA runs its chunks as one sequence across its tiles,
loading the next chunk's fragments under this chunk's MMAs, and the two consumer warpgroups take turns issuing MMAs, so
one warpgroup's epilogue runs while the other's MMAs do.  For every layout, the fused short filter (FIR) and both GELU
transforms, at K of one chunk, a K tail, and 8 and 24 chunks, with a partial last tile, at a small L and at about 2^20
(many tiles per CTA of the persistent grid):
- the result is within the fp64 bar of tests/parity_util.py;
- two runs give the same bits;
- the bits do not depend on which CTA, or which point of the schedule, computed a tile: the call is compared with the
  same rows computed over position ranges (l_range) or, for the GELU variants, which take no range, sample by sample."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_parity import _close, _dev

pytestmark = pytest.mark.gpu

# (act_layout, out_layout, fir, gelu, gelu epilogue)
VARIANTS = {
    "row->ch": (0, 0, False, None, False),
    "row->row": (0, 1, False, None, False),
    "ch->ch": (1, 0, False, None, False),
    "ch->row": (1, 1, False, None, False),
    "ch->row fir": (1, 1, True, None, False),
    "ch->ch fir": (1, 0, True, None, False),
    "gelu tanh prologue": (1, 1, False, "tanh", False),
    "gelu erf prologue": (1, 1, False, "none", False),
    "gelu tanh epilogue": (0, 0, False, "tanh", True),
    "gelu erf epilogue": (0, 0, False, "none", True),
}


def _ref64(act, act_layout, W, out_layout, bias, taps, gelu, pre):
    """fp64 on the device: OUT[b][pos][n] = sum_k A[b][pos][k] W[n][k] (+ bias), with the FIR / GELU transforms."""
    a = act.double()
    if act_layout == 1:
        if taps is not None:
            L = a.shape[-1]
            ap = F.pad(a, (0, 2))
            t = taps.double()
            a = t[:, 2][None, :, None] * ap[..., :L] + t[:, 1][None, :, None] * ap[..., 1:L + 1] \
                + t[:, 0][None, :, None] * ap[..., 2:L + 2]
        if gelu is not None and pre is None:
            a = F.gelu(a, approximate=gelu)
        a = a.transpose(1, 2)
    out = torch.matmul(a, W.double().t())
    if bias is not None:
        out = out + bias.double()
    if pre is not None:
        x = pre.double().requires_grad_(True)
        F.gelu(x, approximate=gelu).sum().backward()
        out = out * x.grad.transpose(1, 2)
    return out if out_layout == 1 else out.transpose(1, 2)


@pytest.mark.parametrize("L", [1000, (1 << 20) - 40])
@pytest.mark.parametrize("K", [32, 100, 256, 768])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_proj_gemm_schedule(variant, K, L):
    import hyena_dna_b200 as H
    dev = _dev()
    act_layout, out_layout, fir, gelu, epi = VARIANTS[variant]
    B = 2 if L < 4096 else 1
    N = 200                                            # a full and a partial tile of outputs
    g = torch.Generator(device=dev).manual_seed(K * 7 + L + len(variant))
    act = torch.randn((B, L, K) if act_layout == 0 else (B, K, L), device=dev, generator=g)
    W = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    bias = None if (gelu is not None or act_layout == 0) else torch.randn(N, device=dev, generator=g)
    taps = torch.randn(K, 3, device=dev, generator=g) if fir else None
    pre = torch.randn(B, N, L, device=dev, generator=g) if epi else None
    kw = {"bias": bias, "fir": taps}
    if gelu is not None:
        kw.update(gelu=gelu, gelu_pre=pre)
    out = H.ops.proj_gemm(act, act_layout, W, False, out_layout, **kw)
    what = f"schedule {variant} K={K} L={L}"
    _close(out, _ref64(act, act_layout, W, out_layout, bias, taps, gelu, pre), what)
    again = H.ops.proj_gemm(act, act_layout, W, False, out_layout, **kw)
    assert torch.equal(out, again), f"{what}: two runs differ in {int((out != again).sum())} elements"
    if gelu is None:
        # rows computed by launches over position ranges whose tiles start elsewhere and run on other CTAs
        pieces = torch.full_like(out, float("nan"))
        cuts = [0, 4 * (L // 12) + 4, 4 * (L // 5), L]
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            H.ops.proj_gemm(act, act_layout, W, False, out_layout, out=pieces, l_range=(lo, hi), **kw)
        assert torch.equal(out, pieces), f"{what}: position ranges differ in {int((out != pieces).sum())} elements"
    elif B > 1:
        for b in range(B):
            one = H.ops.proj_gemm(act[b:b + 1].contiguous(), act_layout, W, False, out_layout, gelu=gelu,
                                  gelu_pre=None if pre is None else pre[b:b + 1].contiguous())
            assert torch.equal(out[b:b + 1], one), f"{what}: sample {b} alone differs"
