"""Projection GEMMs and weight gradients at shapes that exercise the edges of their pipelines, against float64.

The weight-gradient kernel keeps each CTA's running sum in registers for its whole slice of positions and restarts its
accumulator every four chunks; the shapes here give slices shorter than one segment, several segments with a tail, tails of
M, N and L, batch boundaries inside a slice, the hand-staged path (L not a multiple of 4), the fused short filter and both
GELU variants.  The GEMM cases cover K of one and two chunks, several tiles per CTA, the fallback staging path, the fused
prologues and epilogues, and a position-range launch that must leave everything outside its range untouched."""
import pytest
import torch

from tests.test_gpu_parity import _close, _dev

pytestmark = pytest.mark.gpu


def _fir_ref(X, taps):
    """dp[t] = w2 X[t] + w1 X[t+1] + w0 X[t+2] along the last axis (zero beyond the end), float64."""
    L = X.shape[-1]
    Xp = torch.nn.functional.pad(X.double(), (0, 2))
    t = taps.double()
    return t[:, 2][None, :, None] * Xp[..., :L] + t[:, 1][None, :, None] * Xp[..., 1:L + 1] \
        + t[:, 0][None, :, None] * Xp[..., 2:L + 2]


@pytest.mark.parametrize("B,L,M,N", [
    (1, 100, 64, 64),        # four chunks over many splits: every slice is shorter than one segment
    (1, 1000, 200, 136),     # M and N tails, one or two chunks per CTA
    (1, 40000, 200, 136),    # several segments per slice, with a tail segment
    (1, 40001, 128, 128),    # L not a multiple of 4: the producer stages by hand
    (2, 20000, 96, 72),      # slices that cross the batch boundary
])
def test_wgrad_pipeline_matches_fp64(B, L, M, N):
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(B * L + M + N)
    X = torch.randn(B, M, L, generator=g)
    Y = torch.randn(B, L, N, generator=g)
    ref = torch.einsum("bml,bln->mn", X.double(), Y.double())
    _close(H.ops.proj_wgrad(X.to(dev), Y.to(dev)), ref, f"pipeline wgrad {B}x{L}x{M}x{N}")
    _close(H.ops.proj_wgrad(X.to(dev), Y.to(dev), transposed_out=True), ref.t(), f"pipeline wgrad transposed {B}x{L}x{M}x{N}")
    taps = torch.randn(M, 3, generator=g)
    ref_f = torch.einsum("bml,bln->mn", _fir_ref(X, taps), Y.double())
    _close(H.ops.proj_wgrad(X.to(dev), Y.to(dev), fir=taps.to(dev)), ref_f, f"pipeline wgrad FIR {B}x{L}x{M}x{N}")


@pytest.mark.parametrize("approximate", ["tanh", "none"])
def test_wgrad_pipeline_gelu_matches_fp64(approximate):
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(7)
    X = torch.randn(2, 160, 30000, generator=g)
    Y = torch.randn(2, 30000, 72, generator=g)
    gx = torch.nn.functional.gelu(X.double(), approximate=approximate)
    ref = torch.einsum("bml,bln->mn", gx, Y.double())
    _close(H.ops.proj_wgrad(X.to(dev), Y.to(dev), gelu=approximate), ref, f"pipeline wgrad gelu={approximate}")


def test_wgrad_pipeline_is_deterministic():
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(3)
    X = torch.randn(1, 384, 65536, generator=g).to(dev)
    Y = torch.randn(1, 65536, 256, generator=g).to(dev)
    taps = torch.randn(384, 3, generator=g).to(dev)
    a = H.ops.proj_wgrad(X, Y, fir=taps)
    b = H.ops.proj_wgrad(X, Y, fir=taps)
    assert torch.equal(a, b)


@pytest.mark.parametrize("B,L,K,N", [
    (1, 1000, 24, 136),      # one K chunk, N tail
    (2, 777, 40, 200),       # two K chunks, L not a multiple of 4 (fallback staging), batch boundary
    (1, 70000, 256, 384),    # several tiles per CTA
])
def test_proj_gemm_pipeline_matches_fp64(B, L, K, N):
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(B * L + K + N)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    u = torch.randn(B, L, K, generator=g)
    ref = torch.einsum("blk,nk->bnl", u.double(), W.double())
    _close(H.ops.proj_gemm(u.to(dev), 0, W.to(dev), False, 0), ref, f"pipeline gemm row->ch {B}x{L}x{K}x{N}")
    ref_b = torch.einsum("blk,nk->bln", u.double(), W.double()) + bias.double()
    _close(H.ops.proj_gemm(u.to(dev), 0, W.to(dev), False, 1, bias=bias.to(dev)), ref_b,
           f"pipeline gemm row->row bias {B}x{L}x{K}x{N}")
    x = torch.randn(B, K, L, generator=g)
    taps = torch.randn(K, 3, generator=g)
    ref_f = torch.einsum("bkl,nk->bln", _fir_ref(x, taps), W.double())
    _close(H.ops.proj_gemm(x.to(dev), 1, W.to(dev), False, 1, fir=taps.to(dev)), ref_f,
           f"pipeline gemm ch->row FIR {B}x{L}x{K}x{N}")


@pytest.mark.parametrize("approximate", ["tanh", "none"])
def test_proj_gemm_pipeline_gelu_matches_fp64(approximate):
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(11)
    B, L, K, N = 2, 3000, 96, 136
    W = torch.randn(N, K, generator=g) / K ** 0.5
    a = torch.randn(B, K, L, generator=g)
    ref = torch.einsum("bkl,nk->bln", torch.nn.functional.gelu(a.double(), approximate=approximate), W.double())
    _close(H.ops.proj_gemm(a.to(dev), 1, W.to(dev), False, 1, gelu=approximate), ref, f"pipeline gemm gelu={approximate}")
    dy = torch.randn(B, L, K, generator=g)
    pre = torch.randn(B, N, L, generator=g)
    x = pre.double().requires_grad_(True)
    torch.nn.functional.gelu(x, approximate=approximate).sum().backward()
    ref_d = torch.einsum("blk,nk->bnl", dy.double(), W.double()) * x.grad
    _close(H.ops.proj_gemm(dy.to(dev), 0, W.to(dev), False, 0, gelu=approximate, gelu_pre=pre.to(dev)), ref_d,
           f"pipeline gemm dgelu={approximate}")


@pytest.mark.parametrize("act_layout,out_layout,lo,hi", [(0, 0, 1000, 5000), (1, 1, 1000, 5000), (0, 1, 37, 2043),
                                                          (1, 0, 37, 2043)])
def test_proj_gemm_position_range_writes_only_its_range(act_layout, out_layout, lo, hi):
    import hyena_dna_b200 as H
    dev = _dev()
    g = torch.Generator().manual_seed(lo + hi + act_layout)
    B, L, K, N = 2, 6144, 64, 200
    W = torch.randn(N, K, generator=g) / K ** 0.5
    act = torch.randn(B, L, K, generator=g) if act_layout == 0 else torch.randn(B, K, L, generator=g)
    a64 = act.double() if act_layout == 0 else act.double().transpose(1, 2)
    ref = torch.einsum("blk,nk->bln", a64, W.double())
    oshape = (B, N, L) if out_layout == 0 else (B, L, N)
    sentinel = -12345.5
    out = torch.full(oshape, sentinel, device=dev)
    H.ops.proj_gemm(act.to(dev).contiguous(), act_layout, W.to(dev), False, out_layout, out=out, l_range=(lo, hi))
    got = (out if out_layout == 1 else out.transpose(1, 2)).cpu()             # (B, L, N)
    _close(got[:, lo:hi], ref[:, lo:hi], f"pipeline gemm range {act_layout}{out_layout} [{lo}, {hi})")
    outside = torch.cat([got[:, :lo].reshape(-1), got[:, hi:].reshape(-1)])
    assert torch.all(outside == sentinel), "a position-range launch wrote outside its range"
