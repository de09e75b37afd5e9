"""The implicit filter's kernels against fp64: every parameter gradient, at the shapes where the kernels branch.

The filter (csrc/filter_tc.cuh: filter_tc_fwd_kernel, filter_tc_bwd_kernel = backward stage 1, filter_tc_red_kernel =
stage 2; csrc/filter_mlp.cuh behind HYENA_B200_FILTER=simt) picks a code path from L, D, E, the module options and the
size of its sine arguments.  Each test below drives one family of those decisions on purpose and compares k and every
gradient (the eight MLP tensors, dz, ddeltas) with ``filter_ref``, the oracle's filter under fp64 autograd:

| decision                                                         | selected by               | test                                  |
|------------------------------------------------------------------|---------------------------|---------------------------------------|
| 128-position tiles (fwd, stage 1), last partial tile             | L                         | test_sequence_edges                   |
| 32-position K blocks of stage 2, float4 vs scalar loads (L % 4)  | L                         | test_sequence_edges, test_stage2_*    |
| persistent grid: one vs several tiles / K blocks per CTA         | L vs SM count S           | test_sequence_edges[S*128, S*32, ...] |
| output-layer halves (fwd), 64-channel dh.W3 chunks (stage 1),    | D                         | test_channel_edges                    |
|   <= 2 channel tiles (stage 2)                                   |                           |                                       |
| wgmma reduction vs library GEMMs (D <= 256 and E <= 8)           | D, E                      | test_reduction_route                  |
| modulation off, shift != 0, trainable deltas, normalized         | module options            | test_module_options                   |
| z a prefix of a longer embedding (l_max > L), dz                 | lr_pos_emb != 0           | test_z_prefix_of_longer_embedding     |
| inline Cody-Waite sin/cos vs the |x| > 3e4 library branch        | |freq * pre|              | test_sine_arguments                   |
| tensor-core vs CUDA-core filter                                  | HYENA_B200_FILTER=simt    | test_cuda_core_filter (child process) |
| stage 1 on its own (dh and the seven feature-major arrays)       |                           | test_stage1_arrays                    |
| stage 2 on its own: accumulation over 2^20 positions, flush map  | arrays built by the test  | test_stage2_*                         |
| per-(device, stream) grow-only weight images                     | D sequence, two streams   | test_weight_images_across_streams     |

Tail handling is made visible: at long L one position is ~1e-6 of a gradient sum, below any tolerance, so the edge cases
use a ``dk`` that is zero everywhere except the last partial 128-position tile (or the last channel).  Then every gradient
depends on the tail alone.

Comparisons go through tests/parity_util.check: activations with the absolute term scaled by max|ref|, gradients with
``param_grad=True``.  ``filter_ref`` runs twice on the device, in fp64 (the truth, ``ref64``) and in fp32 with TF32 off
(the reference's own numerics, ``ref32``), so the S8(c) hatch can apply and is book-kept.  The tests marked ``gpu`` need
an H100; the reference self-checks at the top run on the CPU.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import hyena_oracle as O
from tests import parity_util as PU

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MLP = ("implicit_filter.0.weight", "implicit_filter.0.bias", "implicit_filter.2.weight", "implicit_filter.2.bias",
       "implicit_filter.4.weight", "implicit_filter.4.bias", "implicit_filter.6.weight", "implicit_filter.1.freq")
GRADS = MLP + ("pos_emb.z", "modulation.deltas")


# ------------------------------------------------------------------------------------------ fp64 reference of the filter
def filter_ref(params, L, dk, dtype=torch.float64, device="cpu", modulate=True, shift=0.0, normalized=False):
    """k (D, L) = O.hyena_filter(L)[0].T and, under the upstream gradient dk (D, L), the gradients of the eight MLP
    tensors, of z (1, l_max, E: zero past L) and of the modulation deltas, keyed by the HyenaFilter parameter names."""
    Q = {n: v.detach().to(device=device, dtype=dtype) for n, v in params.items()}
    for n in GRADS:
        Q["filter_fn." + n] = Q["filter_fn." + n].clone().requires_grad_(True)
    k = O.hyena_filter(L, Q, shift=shift, modulate=modulate, normalized=normalized)[0].t()
    k.backward(dk.to(device=device, dtype=dtype))
    out = {"k": k.detach()}
    for n in GRADS:
        g = Q["filter_fn." + n].grad
        out[n] = g if g is not None else torch.zeros_like(Q["filter_fn." + n])
    return out


def stage1_ref(params, L, dk, dtype=torch.float64, modulate=True, shift=0.0):
    """The arrays backward stage 1 writes, restated: dh (D, L) and a1, a2, a3, dp1, dp2, dp3, X (7, 64, L)."""
    P = {n: v.detach().to(dtype) for n, v in params.items()}
    W = [P[f"filter_fn.implicit_filter.{i}.weight"] for i in (0, 2, 4, 6)]
    b = [P[f"filter_fn.implicit_filter.{i}.bias"] for i in (0, 2, 4)]
    f = P["filter_fn.implicit_filter.1.freq"][0]
    z = P["filter_fn.pos_emb.z"][0, :L]
    t = P["filter_fn.pos_emb.t"][0, :L, 0]
    pre, a = [], []
    h = z
    for l in range(3):
        pre.append(h @ W[l].t() + b[l])
        h = torch.sin(f * pre[-1])
        a.append(h)
    dh = dk.to(dtype)
    if modulate:
        dh = dh * (torch.exp(-t[None, :] * P["filter_fn.modulation.deltas"][0, 0].abs()[:, None]) + shift)
    da = dh.t() @ W[3]
    X = torch.zeros_like(da)
    dp = [None] * 3
    for l in (2, 1, 0):
        g = da * torch.cos(f * pre[l])
        X = X + g * pre[l]
        dp[l] = g * f
        da = dp[l] @ W[l]
    sc = torch.stack([a[0].t(), a[1].t(), a[2].t(), dp[0].t(), dp[1].t(), dp[2].t(), X.t()])
    return dh, sc


def stage2_from_arrays(dh, sc, zT):
    """The parameter gradients as sums over the sequence of the stage-1 arrays (the library route of
    ops._filter_backward_tc, in the arrays' dtype): dW0 = dp1 z, db_l = rowsum(dp_l), dW1 = dp2 a1^T, dW2 = dp3 a2^T,
    dW3 = dh a3^T, dfreq = rowsum(X)."""
    a1, a2, a3, dp1, dp2, dp3, X = sc.unbind(0)
    return dict(dW0=dp1 @ zT.t(), db0=dp1.sum(1), dW1=dp2 @ a1.t(), db1=dp2.sum(1), dW2=dp3 @ a2.t(), db2=dp3.sum(1),
                dW3=dh @ a3.t(), dfreq=X.sum(1))


STAGE2_NAMES = dict(dW0="implicit_filter.0.weight", db0="implicit_filter.0.bias", dW1="implicit_filter.2.weight",
                    db1="implicit_filter.2.bias", dW2="implicit_filter.4.weight", db2="implicit_filter.4.bias",
                    dW3="implicit_filter.6.weight", dfreq="implicit_filter.1.freq")


# ------------------------------------------------------------------------------------------ cases
# Arguments |freq * pre| of the sine layers that straddle the library branch at 3e4 (exactly representable in fp32, so the
# fp32 and fp64 arguments agree and only the sine itself is compared).  test_sine_arguments gives eight features of every
# hidden layer a zero weight row, one of these as bias and freq = 1.
GUARD_ARGS = (100.25, -1000.5, 12345.5, 29999.5, -30000.5, 30000.5, 31415.5, -100000.5)


def case(D, L, E=5, w=10.0, init_std=None, l_max=None, dk="full", seed=0, lr_pos_emb=1e-5, modulate=True, shift=0.0,
         normalized=False, modulation_lr=0.0, guard=False):
    return dict(D=D, L=L, E=E, w=w, init_std=init_std, l_max=l_max or L, dk=dk, seed=seed, lr_pos_emb=lr_pos_emb,
                modulate=modulate, shift=shift, normalized=normalized, modulation_lr=modulation_lr, guard=guard)


def tail_start(L, tile=128):
    """First position of the last (possibly partial) tile."""
    return tile * ((L - 1) // tile)


def case_inputs(c):
    """Seeded host parameters (oracle state_dict keys) and upstream gradient of a case."""
    D, L, E = c["D"], c["L"], c["E"]
    g = torch.Generator().manual_seed(c["seed"])
    P = O.init_params(D, c["l_max"], emb_dim=E, w=c["w"], generator=g, init_std=c["init_std"])
    if c["guard"]:
        n = len(GUARD_ARGS)
        for l, i in enumerate((0, 2, 4)):
            P[f"filter_fn.implicit_filter.{i}.weight"][:n] = 0.0
            P[f"filter_fn.implicit_filter.{i}.bias"][:n] = torch.tensor(GUARD_ARGS[l:] + GUARD_ARGS[:l])
        P["filter_fn.implicit_filter.1.freq"][0, :n] = 1.0
    dk = torch.randn(D, L, generator=g)
    if c["dk"] == "tail":                       # only the last partial tile of 128 (it holds the last K block of 32)
        dk[:, :tail_start(L)] = 0
    elif c["dk"] == "lastch":                   # only the last channel
        dk[:-1] = 0
    elif c["dk"] == "tailw":                    # tail-weighted: a small background everywhere, the tail at full size
        dk[:, :tail_start(L)] *= 0.05
    return P, dk


def make_filter(H, P, c, dev):
    f = H.HyenaFilter(c["D"], emb_dim=c["E"], order=64, seq_len=c["l_max"], w=c["w"], lr_pos_emb=c["lr_pos_emb"],
                      modulate=c["modulate"], normalized=c["normalized"], shift=c["shift"],
                      modulation_lr=c["modulation_lr"])
    sd = {n[len("filter_fn."):]: v for n, v in P.items() if n.startswith("filter_fn.")}
    for extra in ("implicit_filter.3.freq", "implicit_filter.5.freq"):
        sd[extra] = sd["implicit_filter.1.freq"]
    f.load_state_dict(sd, strict=True)
    return f.to(dev)


def expected_grads(c):
    return MLP + (("pos_emb.z",) if c["lr_pos_emb"] else ()) + (("modulation.deltas",) if c["modulation_lr"] else ())


def run_case(H, c, dev):
    """k and the gradients of HyenaFilter.filter_channel_major(L) under dk, as host tensors."""
    P, dk = case_inputs(c)
    f = make_filter(H, P, c, dev)
    k = f.filter_channel_major(c["L"])
    k.backward(dk.to(dev))
    params = dict(f.named_parameters())
    out = {"k": k.detach().cpu()}
    for n in expected_grads(c):
        assert params[n].grad is not None, f"no gradient for {n}"
        out[n] = params[n].grad.cpu()
    return out


def case_refs(c, dev):
    """(fp32 reference, fp64 truth) of a case, both evaluated on dev, returned on the host."""
    P, dk = case_inputs(c)
    opt = dict(modulate=c["modulate"], shift=c["shift"], normalized=c["normalized"])
    r = []
    for dt in (torch.float32, torch.float64):
        o = filter_ref(P, c["L"], dk, dtype=dt, device=dev, **opt)
        r.append({n: v.cpu() for n, v in o.items()})
        del o
        if dev != "cpu":
            torch.cuda.empty_cache()
    return r[0], r[1]


def _act(got, r32, r64, what, s=None):
    """Activation against fp64: absolute term scaled by max|ref| (tests/test_gpu_parity.py::_close)."""
    s = s if s is not None else max(1.0, float(r64.detach().abs().max()))
    return PU.check(got, r32, what + (f" [abs term x{s:.3g}]" if s > 1.0 else ""), ref64=r64, atol=PU.ATOL * s)


def _par(got, r32, r64, what):
    return PU.check(got, r32, what, ref64=r64, param_grad=True)


K_CHUNK = 32                                    # channels of k per comparison (bounds host memory at L = 2^20)


def check_case(tag, c, ours, r32, r64):
    """k (in channel chunks) and every gradient of the case against fp64; returns {name: (|ours-fp64|, |ref32-fp64|)}."""
    errs = {}
    s = max(1.0, float(r64["k"].abs().max()))
    e = [0.0, 0.0]
    for c0 in range(0, c["D"], K_CHUNK):
        sl = slice(c0, c0 + K_CHUNK)
        rec = _act(ours["k"][sl], r32["k"][sl], r64["k"][sl], f"{tag} k[{c0}:{c0 + K_CHUNK}]", s=s)
        e = [max(e[0], rec["e_ours64"]), max(e[1], rec["e_ref64"])]
    errs["k"] = tuple(e)
    for n in expected_grads(c):
        rec = _par(ours[n], r32[n], r64[n], f"{tag} grad {n}")
        errs[n] = (rec["e_ours64"], rec["e_ref64"])
    return errs


def run_and_check(c, tag):
    H = _H()
    dev = _dev()
    ours = run_case(H, c, dev)
    torch.cuda.empty_cache()
    r32, r64 = case_refs(c, dev)
    return check_case(tag, c, ours, r32, r64)


# ------------------------------------------------------------------------------------------ CPU self-checks of the reference
@pytest.mark.parametrize("opt", [dict(), dict(modulate=False), dict(shift=0.25, normalized=True)])
def test_filter_ref_matches_oracle_and_finite_differences(opt):
    """filter_ref's k is O.hyena_filter's, and each of its gradients matches a central finite difference of
    <k, dk> along a random direction of that tensor (L = 40, D = 3, fp64)."""
    D, L, E = 3, 40, 5
    g = torch.Generator().manual_seed(40)
    P = O.to_dtype(O.init_params(D, 48, emb_dim=E, w=10.0, generator=g), torch.float64)
    P["filter_fn.modulation.deltas"] = P["filter_fn.modulation.deltas"] * 30     # visible decay over 40 of 48 positions
    dk = torch.randn(D, L, generator=g, dtype=torch.float64)
    r = filter_ref(P, L, dk, **opt)
    torch.testing.assert_close(r["k"], O.hyena_filter(L, P, **opt)[0].t(), rtol=0, atol=0)
    assert bool((r["pos_emb.z"][:, L:] == 0).all())
    for n in GRADS:
        if n == "modulation.deltas" and opt.get("modulate") is False:
            assert bool((r[n] == 0).all())
            continue
        v = torch.randn(P["filter_fn." + n].shape, generator=g, dtype=torch.float64)
        h = 1e-6
        val = []
        for sgn in (1, -1):
            Q = dict(P)
            Q["filter_fn." + n] = P["filter_fn." + n] + sgn * h * v
            val.append(float((O.hyena_filter(L, Q, **opt)[0].t() * dk).sum()))
        fd = (val[0] - val[1]) / (2 * h)
        an = float((r[n] * v).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), f"{n}: finite difference {fd} vs autograd {an}"


@pytest.mark.parametrize("modulate,shift", [(True, 0.0), (False, 0.0), (True, 0.5)])
def test_stage_refs_compose_to_filter_ref(modulate, shift):
    """stage2_from_arrays(stage1_ref(...)) gives filter_ref's gradients (dz = dp1 W0 too): the restated stage-1 arrays
    and the array -> gradient map the stage-2 tests rely on are the filter's backward."""
    D, L, E = 5, 37, 7
    g = torch.Generator().manual_seed(37)
    P = O.init_params(D, L, emb_dim=E, w=10.0, generator=g)
    dk = torch.randn(D, L, generator=g)
    r = filter_ref(P, L, dk, modulate=modulate, shift=shift)
    dh, sc = stage1_ref(P, L, dk, modulate=modulate, shift=shift)
    zT = P["filter_fn.pos_emb.z"][0, :L].double().t()
    got = stage2_from_arrays(dh, sc, zT)
    for short, n in STAGE2_NAMES.items():
        torch.testing.assert_close(got[short], r[n].reshape(got[short].shape), rtol=1e-10, atol=1e-12, msg=n)
    dz = sc[3].t() @ P["filter_fn.implicit_filter.0.weight"].double()
    torch.testing.assert_close(dz, r["pos_emb.z"][0, :L], rtol=1e-10, atol=1e-12)


def test_parity_bar_rejects_dropped_tail():
    """With a tail-weighted dk (small background, the last partial tile at full size), a result computed without the
    last partial tile -- of dk, or of k itself -- is rejected for k and for every gradient, while the fp64 truth passes."""
    c = case(64, 1000, dk="tailw", seed=5)
    P, dk = case_inputs(c)
    r32, r64 = case_refs(c, "cpu")
    dropped_dk = dk.clone()
    dropped_dk[:, tail_start(c["L"]):] = 0
    bad = filter_ref(P, c["L"], dropped_dk)
    bad_k = r64["k"].clone()
    bad_k[:, tail_start(c["L"]):] = 0
    n0 = len(PU._records)
    try:
        check_case("unperturbed", c, r64, r32, r64)
        with pytest.raises(AssertionError):
            _act(bad_k, r32["k"], r64["k"], "k without its last tile")
        for n in expected_grads(c):
            with pytest.raises(AssertionError):
                _par(bad[n], r32[n], r64[n], f"grad {n} without the last tile of dk")
    finally:
        del PU._records[n0:]            # self-checks of the bar, not parity records


# ------------------------------------------------------------------------------------------ device helpers
def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _H():
    import hyena_dna_b200 as H
    return H


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _length(spec):
    """An L given as an int or as an expression of S, the device's SM count (the persistent grids' size)."""
    return spec if isinstance(spec, int) else int(eval(spec, {"S": _sms()}))


# ------------------------------------------------------------------------------------------ 1. sequence edges
SEQ_L = [1, 2, 127, 128, 129, 255, 31, 32, 33, 34, 4097, "S*128", "S*128+1", "S*32", "S*32+1", (1 << 20) - 3]


@gpu
@pytest.mark.parametrize("L", SEQ_L)
def test_sequence_edges(L):
    """Tiles of 128 positions (forward, stage 1) with a partial last tile; K blocks of 32 (stage 2) with float4 or scalar
    loads; one or several tiles / K blocks per CTA of the persistent grids.  D = 256 (two output halves, four dh.W3 chunks,
    two channel tiles); dk lives on the last partial tile only, so every gradient is the tail's."""
    L = _length(L)
    run_and_check(case(256, L, dk="tail", seed=L), f"seq L={L}")


# ------------------------------------------------------------------------------------------ 2. channel edges
SEQ_D = [1, 8, 63, 64, 65, 127, 128, 129, 192, 255, 256]


@gpu
@pytest.mark.parametrize("dk", ["full", "lastch"])
@pytest.mark.parametrize("D", SEQ_D)
def test_channel_edges(D, dk):
    """Output-layer halves of 128 channels, 64-channel chunks of dh.W3, one or two channel tiles of stage 2, each with a
    partial last part; "lastch": dk on the last channel only, so the gradients are that channel's alone."""
    run_and_check(case(D, 1000, dk=dk, seed=1000 + D), f"channels D={D} dk={dk}")


# ------------------------------------------------------------------------------------------ 3. reduction route
@gpu
@pytest.mark.parametrize("D,E", [(257, 5), (320, 5), (512, 5), (64, 9), (256, 15), (256, 3), (256, 7), (200, 7)])
def test_reduction_route(D, E):
    """Stage 2 on filter_tc_red_kernel (D <= 256 and E <= 8) or on the library GEMMs; the profiler shows which ran."""
    H = _H()
    H._lib.profile_begin()
    run_and_check(case(D, 4097, E=E, seed=D + E), f"route D={D} E={E}")
    prof = H._lib.profile_end()
    assert ("filter_tc_red" in prof) == (D <= 256 and E <= 8), prof
    assert "filter_tc_bwd" in prof and "filter_tc_fwd" in prof, prof


# ------------------------------------------------------------------------------------------ 4. module options
OPTIONS = {"modulation_off": dict(modulate=False), "shift": dict(shift=0.25),
           "trainable_deltas": dict(modulation_lr=1e-3), "normalized": dict(normalized=True)}


@gpu
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_module_options(opt):
    """Modulation off, shift != 0, trainable deltas (filter_ddelta_kernel), L1-normalised filter (l1norm_*), at the
    BASELINE width D = 256 and L = 40000."""
    run_and_check(case(256, 40000, seed=40000, **OPTIONS[opt]), f"option {opt}")


@gpu
def test_z_prefix_of_longer_embedding():
    """The filter of L = 20011 positions of an embedding of l_max = 32768: dz covers the prefix, zero past it."""
    errs = run_and_check(case(256, 20011, l_max=32768, seed=20011), "z prefix L=20011 l_max=32768")
    assert "pos_emb.z" in errs


# ------------------------------------------------------------------------------------------ 5. sine arguments
@gpu
@pytest.mark.parametrize("w,init_std", [(1.0, None), (10.0, None), (100.0, 0.005), ("guard", None)])
def test_sine_arguments(w, init_std):
    """freq * pre-activation grows with w: unit-scale init at w = 1 and 10 (arguments up to ~1e2).  At w = 100 the
    MLP is ill-conditioned in fp32 unless its weights are small (the reference's own fp32 filter is 4e-3 normwise from
    fp64 with unit-scale init, 41 % of its elements miss the bound; 3e-5 with init 0.02), so that case uses init 0.005.
    "guard": eight features of every hidden layer get exactly
    representable arguments from 100 to 1e5 (GUARD_ARGS), so the inline reduction up to 3e4 and the library branch past
    it are compared with the exact sine."""
    if w == "guard":
        c = case(64, 4097, w=10.0, guard=True, seed=3)
    else:
        c = case(64, 4097, w=w, init_std=init_std, seed=int(w))
    run_and_check(c, f"sine w={w} init={init_std or 'unit'}")


# ------------------------------------------------------------------------------------------ 6. CUDA-core filter
SIMT_CASES = {
    "seq": case(256, 4097, dk="tail", seed=11),
    "channels": case(129, 1000, dk="lastch", seed=12),
    "wide": case(320, 1500, seed=13),
    "options": case(256, 40000, shift=0.25, modulation_lr=1e-3, seed=14),
    "guard": case(64, 4097, guard=True, seed=15),
}


def simt_child(path):
    """Entry point of the child process (HYENA_B200_FILTER=simt is read once per process by the forward)."""
    import numpy as np
    H = _H()
    dev = _dev()
    H._lib.profile_begin()
    arrs = {}
    for name, c in SIMT_CASES.items():
        for n, v in run_case(H, c, dev).items():
            arrs[f"{name}|{n}"] = v.numpy()
    prof = H._lib.profile_end()
    arrs["kinds"] = np.array(sorted(prof))
    np.savez(path, **arrs)


@gpu
def test_cuda_core_filter(tmp_path):
    """The CUDA-core filter (csrc/filter_mlp.cuh) in a child process with HYENA_B200_FILTER=simt: no tensor-core filter
    kernel runs, and k and every gradient of the core cases match fp64."""
    import numpy as np
    dev = _dev()
    out = tmp_path / "simt.npz"
    env = dict(os.environ, HYENA_B200_FILTER="simt")
    code = f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_gpu_filter_paths import simt_child; simt_child({str(out)!r})"
    res = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    z = np.load(out)
    kinds = set(z["kinds"].tolist())
    assert {"filter_fwd", "filter_bwd"} <= kinds, kinds
    assert not any(k.startswith("filter_tc") for k in kinds), kinds
    for name, c in SIMT_CASES.items():
        ours = {n: torch.from_numpy(z[f"{name}|{n}"]) for n in ("k",) + expected_grads(c)}
        r32, r64 = case_refs(c, dev)
        check_case(f"simt {name}", c, ours, r32, r64)


# ------------------------------------------------------------------------------------------ 7. full size
@gpu
@pytest.mark.parametrize("init_std", [0.02, None])
def test_full_size(init_std):
    """D = 256, L = 2^20, E = 5, w = 10, trainable deltas and z: k and all ten gradients against fp64; prints, per tensor,
    max|ours - fp64| next to max|fp32 ref - fp64|."""
    c = case(256, 1 << 20, init_std=init_std, modulation_lr=1e-3, seed=20)
    errs = run_and_check(c, f"full size init={init_std or 'unit'}")
    print(f"\nfull size D=256 L=2^20 E=5 w=10 init={init_std or 'unit'}: max|ours - fp64| vs max|fp32 ref - fp64|")
    for n, (eo, er) in errs.items():
        print(f"  {n:28s} {eo:.3e}  {er:.3e}")


# ------------------------------------------------------------------------------------------ 8. stage 1 on its own
def _mlp_args(f):
    m = f.implicit_filter
    return [a.detach() for a in (f.pos_emb.z, f.pos_emb.t, m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight,
                                 m[4].bias, m[6].weight, m[1].freq, f.modulation.deltas)]


def _k_and_stage1(H, f, L, dk):
    """ops.filter_forward and backward stage 1 on the current stream: k (D, L), dh (D, L), the seven arrays (7, 64, L)."""
    args = _mlp_args(f)
    shift, mod = float(f.modulation.shift), bool(f.modulate)
    k = H.ops.filter_forward(*args, shift, mod, L)
    zz, tt, E, N, D = H.ops._filter_args(*args, shift, mod, L)
    ws = [x.contiguous() for x in args[2:9]]
    fr, dl = args[9].reshape(-1).contiguous(), args[10].reshape(-1).contiguous()
    dh = torch.empty(D, L, device=dk.device)
    sc = torch.empty(7, 64, L, device=dk.device)
    H._lib.check(H._lib.lib().hyena_b200_filter_bwd_stage1(
        zz.data_ptr(), zz.stride(0), tt.data_ptr(), *[w.data_ptr() for w in ws], fr.data_ptr(), dl.data_ptr(), shift,
        int(mod), L, E, N, D, dk.data_ptr(), dh.data_ptr(), sc.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return k, dh, sc


@gpu
@pytest.mark.parametrize("D,L", [(65, 129), (256, 4097), (192, 40000)])
def test_stage1_arrays(D, L):
    """dh and a1, a2, a3, dp1, dp2, dp3, X from filter_tc_bwd_kernel against stage1_ref in fp32 and fp64.  w = 1: at w = 10
    with unit-scale init the fp32 sines are ~2e-5 from fp64 (either implementation), too far for an elementwise bound on
    activations of unit size; k and the gradients average that out."""
    H = _H()
    dev = _dev()
    c = case(D, L, w=1.0, seed=D * L)
    P, dk = case_inputs(c)
    f = make_filter(H, P, c, dev)
    _, dh, sc = _k_and_stage1(H, f, L, dk.to(dev))
    r32 = stage1_ref(P, L, dk, dtype=torch.float32)
    r64 = stage1_ref(P, L, dk)
    _act(dh, r32[0], r64[0], f"stage 1 D={D} L={L} dh")
    for i, n in enumerate(("a1", "a2", "a3", "dp1", "dp2", "dp3", "X")):
        _act(sc[i], r32[1][i], r64[1][i], f"stage 1 D={D} L={L} {n}")


# ------------------------------------------------------------------------------------------ 9. stage 2 on its own
# The tensor core adds into its accumulator with truncation.  filter_tc_red_kernel used to chain all MMAs of a CTA's K blocks
# into one accumulator: on same-sign arrays at L = 2^20 that put dW0 8.5e-5 (relative to max|fp64|) off, 110x the fp32
# library route.  It now restarts every 8 blocks and flushes with atomic adds, whose own rounding (132 CTAs x ~30 flushes
# into every element) keeps it a few times above the library.  The bound: STAGE2_FACTOR times the error of the fp32 library
# route on the same arrays (cuBLAS, TF32 off: the route wide models take), with a floor of 2^-20 max|fp64| for sums the
# library gets exactly (one-hot rows).
STAGE2_FACTOR = 10.0


def stage2_arrays(kind, D, E, L, seed):
    """dh (D, L), the seven arrays (7, 64, L) and zT (E, L) on the device.  "random": N(0, 1); "same_sign": U(0, 1), no
    cancellation, so a truncation bias accumulates coherently; "onehot": a3, a2, a1 and z rows each hold a single 1 (at a
    distinct position, first and last included), so every element of dW3, dW2, dW1 and dW0 is one element of dh, dp3,
    dp2, dp1 and a flush to a wrong place cannot cancel out."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = torch.device("cuda:0")
    if kind == "same_sign":
        dh = torch.rand(D, L, generator=g, device=dev)
        sc = torch.rand(7, 64, L, generator=g, device=dev)
        zT = torch.rand(E, L, generator=g, device=dev)
    else:
        dh = torch.randn(D, L, generator=g, device=dev)
        sc = torch.randn(7, 64, L, generator=g, device=dev)
        zT = torch.randn(E, L, generator=g, device=dev)
    if kind == "onehot":
        pos = torch.randperm(L, generator=torch.Generator().manual_seed(seed))
        pos = torch.cat([torch.tensor([L - 1, 0]), pos[(pos != 0) & (pos != L - 1)]])
        for j, arr in enumerate((0, 1, 2)):                  # a1, a2, a3
            sc[arr].zero_()
            p = pos[(64 * j + torch.arange(64)) % L].to(dev)
            sc[arr, torch.arange(64, device=dev), p] = 1.0
        zT.zero_()
        p = pos[(192 + torch.arange(E)) % L].to(dev)
        zT[torch.arange(E, device=dev), p] = 1.0
    return dh, sc, zT


def _stage2(H, dh, sc, zT):
    D, L = dh.shape
    E = zT.shape[0]
    dev = dh.device
    o = dict(dW0=torch.zeros(64, E, device=dev), db0=torch.zeros(64, device=dev), dW1=torch.zeros(64, 64, device=dev),
             db1=torch.zeros(64, device=dev), dW2=torch.zeros(64, 64, device=dev), db2=torch.zeros(64, device=dev),
             dW3=torch.zeros(D, 64, device=dev), dfreq=torch.zeros(64, device=dev))
    H._lib.check(H._lib.lib().hyena_b200_filter_bwd_stage2(
        dh.data_ptr(), sc.data_ptr(), zT.data_ptr(), *[o[n].data_ptr() for n in ("dW0", "db0", "dW1", "db1", "dW2", "db2",
                                                                                  "dW3", "dfreq")],
        L, E, D, torch.cuda.current_stream().cuda_stream))
    return o


def check_stage2(kind, D, E, L, seed):
    H = _H()
    _dev()
    dh, sc, zT = stage2_arrays(kind, D, E, L, seed)
    ours = _stage2(H, dh, sc, zT)
    lib = stage2_from_arrays(dh, sc, zT)
    r64 = stage2_from_arrays(dh.double(), sc.double(), zT.double())
    tag = f"stage 2 {kind} D={D} E={E} L={L}"
    rows = []
    for n in r64:
        scale = float(r64[n].abs().max())
        e_ours = float((ours[n].double() - r64[n]).abs().max())
        e_lib = float((lib[n].double() - r64[n]).abs().max())
        rows.append((n, e_ours, e_lib, scale))
    print(f"\n{tag}: max error / max|fp64|, ours vs fp32 library")
    for n, eo, el, scale in rows:
        print(f"  {n:6s} {eo / scale:.2e}  {el / scale:.2e}")
    for n, eo, el, scale in rows:
        _par(ours[n], lib[n], r64[n], f"{tag} {n}")
        bound = STAGE2_FACTOR * max(el, 2.0 ** -20 * scale)
        assert eo <= bound, (f"{tag} {n}: max|ours - fp64| = {eo:.3e} ({eo / scale:.2e} of max|fp64|) exceeds "
                             f"{STAGE2_FACTOR} x max(library fp32 error {el:.3e}, 2^-20 max|fp64|)")


@gpu
@pytest.mark.parametrize("kind", ["random", "same_sign", "onehot"])
@pytest.mark.parametrize("L", [33, 4097, "S*32+1", 1 << 20])
def test_stage2_data(kind, L):
    """Random, same-sign and one-hot arrays at D = 256, E = 5, up to L = 2^20."""
    L = _length(L)
    check_stage2(kind, 256, 5, L, seed=L)


@gpu
@pytest.mark.parametrize("E", [1, 2, 3, 4, 5, 6, 7, 8])
def test_stage2_every_emb_dim(E):
    """The ABI takes E = 1..8 (not only odd E): the z rows of G3 and the dW0 / db0 columns."""
    check_stage2("onehot", 129, E, 4099, seed=E)
    check_stage2("random", 129, E, 4099, seed=10 + E)


# ------------------------------------------------------------------------------------------ 10. bar tight enough
@gpu
def test_parity_bar_rejects_tf32_reference():
    """The fp32 reference with TF32 on (one MMA per product instead of 3xTF32) is rejected at D = 256, L = 40000, for k
    and for the output-layer weight gradient, while the fp64 truth passes."""
    dev = _dev()
    c = case(256, 40000, seed=41)
    P, dk = case_inputs(c)
    r32, r64 = case_refs(c, dev)
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        tf = filter_ref(P, c["L"], dk, dtype=torch.float32, device=dev)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    tf = {n: v.cpu() for n, v in tf.items()}
    n0 = len(PU._records)
    try:
        _act(r64["k"], r32["k"], r64["k"], "fp64 truth k")
        with pytest.raises(AssertionError):
            _act(tf["k"], r32["k"], r64["k"], "TF32 reference k")
        with pytest.raises(AssertionError):
            _par(tf["implicit_filter.6.weight"], r32["implicit_filter.6.weight"], r64["implicit_filter.6.weight"],
                 "TF32 reference grad implicit_filter.6.weight")
    finally:
        del PU._records[n0:]


# ------------------------------------------------------------------------------------------ 11. streams and determinism
@gpu
def test_weight_images_across_streams():
    """The weight images are per (device, stream) and only grow.  k, dh and the seven stage-1 arrays are bitwise equal to
    an isolated run after D = 64 -> 320 -> 64 on one stream, when two streams interleave, and across repeats.  The
    stage-2 gradients use atomics, so they are held to the fp64 tolerance only."""
    H = _H()
    dev = _dev()
    L = 40000
    cs = {D: case(D, L, seed=D) for D in (64, 320)}
    inp = {D: case_inputs(c) for D, c in cs.items()}
    fs = {D: make_filter(H, inp[D][0], cs[D], dev) for D in cs}
    dks = {D: inp[D][1].to(dev) for D in cs}

    def run(D):
        return [t.clone() for t in _k_and_stage1(H, fs[D], L, dks[D])]

    def same(a, b, what):
        for n, x, y in zip(("k", "dh", "stage-1 arrays"), a, b):
            assert torch.equal(x, y), f"{what}: {n} differs"

    base = {}
    for D in (64, 320):
        base[D] = run(D)
        torch.cuda.synchronize()
        same(run(D), base[D], f"D={D} repeat")
    for D in (64, 320, 64):
        same(run(D), base[D], f"D={D} in the sequence 64, 320, 64")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    got = []
    for D, s in ((64, s1), (320, s2), (320, s1), (64, s2), (64, s1)):
        with torch.cuda.stream(s):
            got.append((D, run(D)))
    torch.cuda.synchronize()
    for i, (D, o) in enumerate(got):
        same(o, base[D], f"D={D} interleaved on two streams (call {i})")
    grads = {}
    for D, s in ((64, s1), (320, s2)):
        with torch.cuda.stream(s):
            k = fs[D].filter_channel_major(L)
            k.backward(dks[D])
    torch.cuda.synchronize()
    for D in cs:
        params = dict(fs[D].named_parameters())
        r32, r64 = case_refs(cs[D], dev)
        for n in expected_grads(cs[D]):
            _par(params[n].grad, r32[n], r64[n], f"two streams D={D} grad {n}")
