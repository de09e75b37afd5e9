"""Packed prompts into a decode cache (``prefill`` / ``admit`` with ``cu_seqlens=``; hyena_b200_decode_admit_packed;
DESIGN.md section 4.19) without a GPU: the C entry point's guards, the host checks of HyenaOperator, Block and Backbone,
each firing before any device work, and a self-check that the per-sequence decode truth the GPU tests use rejects a cache
filled with planted placement bugs."""
import ctypes
from functools import partial
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from oracle import hyena_oracle as O
from tests import parity_util as PU
from tests.test_decode_admit_cpu import _cpu_cache

_lib = import_module("hyena_dna_b200._lib")

PTR = ctypes.c_void_p(256)          # never dereferenced: the checks come first


def _err():
    return _lib.lib().hyena_b200_last_error().decode()


def _H():
    import hyena_dna_b200 as H
    return H


# ---------------------------------------------------------------------------------------------- helpers of the GPU tests
def decode_truth(prompts, conts, P, dtype, device=None):
    """Truth of decoding after packed prompts: the oracle on each whole sequence (prompt i then conts[i]) alone, in
    ``dtype`` on ``device`` -> [outputs (m_i, D) at the continuation's positions]."""
    device = device or torch.device("cpu")
    Q = {k: v.to(device, dtype) for k, v in P.items()}
    out = []
    for x, c in zip(prompts, conts):
        seq = torch.cat([x, c]).to(device, dtype)[None]
        out.append(O.hyena_operator(seq, Q)[0, x.shape[0]:])
    return out


# ---------------------------------------------------------------------------------------------- C entry point
def test_abi_present_and_no_new_kinds():
    L = _lib.lib()
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "hyena_b200.h")) as f:
        header = f.read()
    for name in ("hyena_b200_decode_admit_packed", "hyena_b200_decode_admit_packed_h16"):
        assert name in _lib.SIGNATURES and hasattr(L, name) and name + "(" in header
    assert L.hyena_b200_abi_version() == 3 and L.hyena_b200_kind_count() == 33


def _admit_packed(p=PTR, h=PTR, tail=PTR, rows=PTR, sg=PTR, rs=PTR, ib=None, T=100, k=2, cache_B=4, order=2, Pn=16,
                  t=32, Lcap=64, code=None):
    args = (p, ib, PTR, PTR, h, tail, rows, sg, rs, T, k, cache_B, 8, order, Pn, t, Lcap, None)
    if code is None:
        return _lib.lib().hyena_b200_decode_admit_packed(*args)
    return _lib.lib().hyena_b200_decode_admit_packed_h16(code, *args)


GUARDS = [(dict(p=None), "null pointer"), (dict(h=None), "null pointer"), (dict(tail=None), "null pointer"),
          (dict(rows=None), "null pointer"), (dict(sg=None), "null pointer"), (dict(rs=None), "null pointer"),
          (dict(k=5), "5 prompts"), (dict(k=0), "bad shape"), (dict(order=1), "order"), (dict(order=32), "order"),
          (dict(Lcap=(1 << 20) + 4, t=8), "exceeds"), (dict(Pn=33), "cannot end"), (dict(Pn=0), "cannot end"),
          (dict(t=65), "outside the decode cache"), (dict(T=0), "bad packed length"), (dict(T=15), "bad packed length"),
          (dict(p=ctypes.c_void_p(258)), "misaligned"), (dict(rows=ctypes.c_void_p(258)), "misaligned"),
          (dict(rs=ctypes.c_void_p(258)), "misaligned"), (dict(sg=ctypes.c_void_p(260)), "misaligned"),
          (dict(ib=ctypes.c_void_p(258)), "misaligned")]


@pytest.mark.parametrize("code", [None, _lib.HIST_F16, _lib.HIST_BF16])
def test_decode_admit_packed_guards(code):
    n0 = _lib.launch_count()
    for kw, msg in GUARDS:
        assert _admit_packed(code=code, **kw) != 0 and msg in _err(), (code, kw, _err())
    assert _admit_packed(code=7) != 0 and "unknown history dtype" in _err()
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- host checks first
@pytest.fixture
def no_device(monkeypatch):
    """Every device entry point of a packed prefill or admission fails the test if reached."""
    H = _H()
    for name in ("core_forward_packed", "decode_admit_packed", "decode_admit", "decode_hist", "decode_shift", "proj_gemm",
                 "add_layer_norm", "filter_spectrum", "packed_plan"):
        monkeypatch.setattr(H.ops, name, lambda *a, _n=name, **k: pytest.fail(f"device work ({_n}) before validation"))
    return H


def _cu(*n):
    out = [0]
    for x in n:
        out.append(out[-1] + x)
    return torch.tensor(out)


# (keywords of the call, the cache, the expected message); the prefill cache has 2 rows, the admission cache 4 rows at t
PREFILL = [(dict(cu=_cu(3, 5, 2)), {}, "3 packed prompts for a decode cache of 2 rows"),
           (dict(cu=_cu(8, 0)), {}, "prompt 1 is empty"),
           (dict(cu=_cu(40, 30)), dict(lcap=32), "exceeds Lcap = 32"),
           (dict(cu=_cu(65, 5)), {}, "exceeds l_max"),
           (dict(cu=_cu(6, 4), max_seqlen=5), {}, "max_seqlen = 5 is shorter"),
           (dict(cu=_cu(6, 4), lengths=[6, 4]), {}, "does not combine with lengths"),
           (dict(cu=_cu(6, 4), grad=True), {}, "requires grad"),
           (dict(cu=_cu(6, 4)), dict(t=8), "fresh cache; this one is at position 8"),
           (dict(cu=_cu(6, 4)), dict(branched=True), "branched"),
           (dict(cu=torch.tensor([1, 6, 10])), {}, r"cu_seqlens\[0\] must be 0"),
           (dict(cu=torch.tensor([0, 7, 6, 10])), {}, "non-decreasing"),
           (dict(cu=torch.tensor([0, 6, 11]), shape=(10, 8)), {}, "must equal the number of packed positions"),
           (dict(cu=torch.tensor([0.0, 10.0])), {}, "integer"),
           (dict(cu=_cu(6, 4), shape=(2, 5, 8)), {}, "packed input")]
ADMIT = [(dict(cu=_cu(3, 5), rows=[0, 4]), {}, r"rows 4 outside \[0, 4\)"),
         (dict(cu=_cu(3, 5), rows=[1, 1]), {}, "repeat"),
         (dict(cu=_cu(3, 5), rows=[2]), {}, "1 rows for 2 packed prompts"),
         (dict(cu=_cu(3, 5, 2), rows=[0, 1]), {}, "2 rows for 3 packed prompts"),
         (dict(cu=_cu(3, 0), rows=[0, 1]), {}, "prompt 1 is empty"),
         (dict(cu=_cu(3, 64), rows=[0, 1]), dict(lcap=60), "exceeds Lcap"),
         (dict(cu=_cu(3, 65), rows=[0, 1]), {}, "exceeds l_max"),
         (dict(cu=_cu(3, 63), rows=[0, 1]), dict(t=41), "right shift"),
         (dict(cu=_cu(3, 5), rows=[0, 1], lengths=[3, 5]), {}, "does not combine with lengths"),
         (dict(cu=_cu(3, 5), rows=[0, 1], grad=True), {}, "requires grad"),
         (dict(cu=_cu(3, 5), rows=[0, 1]), dict(branched=True), "branched"),
         (dict(cu=torch.tensor([0, 5, 3, 8]), rows=[0, 1]), {}, "non-decreasing")]


def _cases(how, order=2, bidirectional=False):
    H = _H()
    mk = partial(H.HyenaOperator, l_max=64, emb_dim=5, order=order, bidirectional=bidirectional)
    return H, mk(8), H.Block(8, mixer_cls=mk), H.Backbone(8, 2, mk)


def _run_all(H, op, block, bb, kw, cache_kw, how, msg):
    total = int(kw["cu"][-1])
    u = torch.zeros(kw.get("shape", (total, 8)), requires_grad=kw.get("grad", False))
    B = 2 if how == "prefill" else 4

    def cache(m):
        c = _cpu_cache(m, B=B, lcap=cache_kw.get("lcap", 64), t=cache_kw.get("t", 0 if how == "prefill" else 20))
        c._branched = cache_kw.get("branched", False)
        return c
    extra = {k: kw[k] for k in ("lengths",) if k in kw}
    if how == "prefill":
        if "max_seqlen" in kw:
            extra["max_seqlen"] = kw["max_seqlen"]
        calls = [lambda: op.prefill(u, cache(op), cu_seqlens=kw["cu"], **extra),
                 lambda: block.prefill(u, None, cache(block.mixer), cu_seqlens=kw["cu"], **extra),
                 lambda: bb.prefill(u, H.DecodeCache.stack([cache(la.mixer) for la in bb.layers]), cu_seqlens=kw["cu"],
                                    **extra)]
    else:
        rows = kw["rows"]
        calls = [lambda: op.admit(u, cache(op), rows, cu_seqlens=kw["cu"], **extra),
                 lambda: block.admit(u, None, cache(block.mixer), rows, cu_seqlens=kw["cu"], **extra),
                 lambda: bb.admit(u, H.DecodeCache.stack([cache(la.mixer) for la in bb.layers]), rows,
                                  cu_seqlens=kw["cu"], **extra)]
    n0 = H.launch_count()
    for call in calls:
        with pytest.raises(H.HyenaB200Error, match=msg):
            call()
    assert H.launch_count() == n0


@pytest.mark.parametrize("i", range(len(PREFILL)))
def test_packed_prefill_checks_run_before_device_work(no_device, i):
    kw, cache_kw, msg = PREFILL[i]
    _run_all(*_cases("prefill"), kw, cache_kw, "prefill", msg)


@pytest.mark.parametrize("i", range(len(ADMIT)))
def test_packed_admit_checks_run_before_device_work(no_device, i):
    kw, cache_kw, msg = ADMIT[i]
    _run_all(*_cases("admit"), kw, cache_kw, "admit", msg)


@pytest.mark.parametrize("how", ["prefill", "admit"])
@pytest.mark.parametrize("variant,msg", [(dict(order=3), "order 2"), (dict(bidirectional=True), "bidirectional")])
def test_packed_decoding_needs_order_2_and_a_causal_filter(no_device, how, variant, msg):
    H = _H()
    kw = dict(cu=_cu(6, 4)) if how == "prefill" else dict(cu=_cu(6, 4), rows=[0, 1])
    _run_all(*_cases(how, **variant), kw, {}, how, msg)


def test_valid_packed_calls_reach_the_device_check(no_device):
    """Every check passes: the next thing is the device, and a CPU input stops there."""
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    n0 = H.launch_count()
    with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
        op.prefill(torch.zeros(1, 10, 8), _cpu_cache(op, B=2), cu_seqlens=_cu(6, 4), max_seqlen=6)
    for t, n in ((20, (3, 5)), (0, (8, 1)), (3, (1, 60)), (64, (64, 2))):
        with pytest.raises(H.HyenaB200Error, match="no CPU fallback"):
            op.admit(torch.zeros(sum(n), 8), _cpu_cache(op, t=t), torch.tensor([2, 0]), cu_seqlens=_cu(*n))
    assert H.launch_count() == n0


def test_forward_with_a_decode_cache_still_raises(no_device):
    H = _H()
    op = H.HyenaOperator(8, 64, emb_dim=5)
    with pytest.raises(H.HyenaB200Error, match="DecodeCache.*prefill.*cu_seqlens"):
        op(torch.zeros(10, 8), cu_seqlens=_cu(6, 4), inference_params=_cpu_cache(op, B=2))
    for how in (op.step, op.extend):
        with pytest.raises(TypeError):
            how(torch.zeros(2, 1, 8), _cpu_cache(op, B=2), cu_seqlens=_cu(1, 1))


# ---------------------------------------------------------------------------------------------- truth self-check
def _decode_model(prompts, conts, P, bug=None):
    """fp64 model of decoding from a cache filled with the packed prompts, with one planted bug: "early" places each
    prompt's history one position early (a zero position between it and the continuation), "tail" fills the tail of a
    one-position prompt with the previous prompt's last position where it should hold a pad (0), "start" puts each row's
    start one position late (the prompt's first position becomes padding) -> [outputs at the continuation's positions]."""
    Q = O.to_dtype(P, torch.float64)
    D = prompts[0].shape[1]
    out = []
    for i, (x, c) in enumerate(zip(prompts, conts)):
        n = x.shape[0]
        seq = torch.cat([x, c]).double()
        p = F.linear(seq, Q["in_proj.weight"], Q["in_proj.bias"]).T[None]           # (1, 3D, L)
        if bug == "start":
            p[..., 0] = 0.0
        uc = O.short_filter(p, Q["short_filter.weight"], Q["short_filter.bias"], p.shape[-1])
        if bug == "tail" and i > 0:                     # the prompt's own positions are right; the first step reads the tail
            prev = F.linear(prompts[i - 1][-1:].double(), Q["in_proj.weight"], Q["in_proj.bias"]).T[None]
            pp = torch.cat([prev, p], -1)
            uc[..., n:] = O.short_filter(pp, Q["short_filter.weight"], Q["short_filter.bias"], pp.shape[-1])[..., n + 1:]
        x0, x1, v = uc.split(D, dim=1)
        g = v * x1
        if bug == "start":
            g[..., 0] = 0.0
        L = g.shape[-1] + 1
        k = O.hyena_filter(L, Q)[0].T                                                   # (D, L)
        fb = Q["filter_fn.bias"].reshape(-1)
        if bug == "early":
            ge = torch.cat([g[..., :n], torch.zeros_like(g[..., :1]), g[..., n:]], -1)
            conv = O.fftconv_ref(ge, k, 0 * fb)[..., 1:]
            conv[..., :n] = O.fftconv_ref(g, k[:, :L - 1], 0 * fb)[..., :n]
            y_pre = (conv + fb[:, None] * g) * x0
        else:
            y_pre = O.fftconv_ref(g, k[:, :L - 1], fb) * x0
        y = F.linear(y_pre[0].T, Q["out_proj.weight"], Q["out_proj.bias"])
        out.append(y[n:])
    return out


@pytest.mark.parametrize("bug", ["early", "tail", "start"])
def test_decode_truth_rejects_planted_bugs(bug):
    D = 4
    g = torch.Generator().manual_seed(3)
    P = O.init_params(D, 64, emb_dim=5, w=10.0, generator=g, init_std=0.1)        # outputs well above out_proj.bias
    P["in_proj.bias"] = 0.1 * torch.randn(P["in_proj.bias"].shape, generator=g)
    lengths, m = [5, 1, 9, 1], 6
    prompts = [O.nucleotide_activations(1, n, D, seed=40 + i)[0][0] for i, n in enumerate(lengths)]
    conts = [O.nucleotide_activations(1, m, D, seed=60 + i)[0][0] for i in range(len(lengths))]
    t32 = decode_truth(prompts, conts, P, torch.float32)
    t64 = decode_truth(prompts, conts, P, torch.float64)
    good = _decode_model(prompts, conts, P)
    for i in range(len(lengths)):                       # the model without a bug meets the bar
        PU.check(good[i], t32[i], f"decode model seq {i}", ref64=t64[i])
    bad = _decode_model(prompts, conts, P, bug)
    missed = 0
    hit = [i for i in range(len(lengths)) if bug != "tail" or (i > 0 and lengths[i] == 1)]
    for i in hit:
        try:
            PU.check(bad[i], t32[i], f"planted {bug} seq {i}", ref64=t64[i])
        except AssertionError:
            missed += 1
    PU._records[:] = [r for r in PU._records if not r["what"].startswith("planted")]
    assert missed == len(hit) and len(hit) >= 2, f"the bar let a planted {bug} bug through"
