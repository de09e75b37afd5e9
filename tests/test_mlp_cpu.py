"""Block MLP (hyena_dna_b200.Mlp) without a GPU: reference state_dict layout, constructor guards, no CPU fallback, and the
sm_90a build of the fused-GELU projection kernels.

tests/golden/ref_mlp_keys.json is written by tests/golden/make_mlp_keys.py from the UNMODIFIED reference
flash_attn.modules.mlp.Mlp; tests/golden/ref_model_keys.json holds the keys of the reference whole model."""
import json
import os
import re
import shutil
import subprocess
from functools import partial

import pytest
import torch
import torch.nn.functional as F

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _shapes(module):
    return {k: list(v.shape) for k, v in module.state_dict().items()}


def test_state_dict_matches_reference_mlp():
    import hyena_dna_b200 as H
    with open(os.path.join(GOLD, "ref_mlp_keys.json")) as f:
        cases = json.load(f)
    assert any(c["kwargs"].get("bias1") is False for c in cases) and any(c["kwargs"].get("bias2") is False for c in cases)
    for c in cases:
        assert _shapes(H.Mlp(**c["kwargs"])) == c["keys"], c["kwargs"]


def test_reference_checkpoint_mlp_keys_load():
    """create_mlp_cls (long_conv_lm.py:102-123) = partial(Mlp, hidden_features=d_inner, activation=gelu tanh): the
    backbone.layers.N.mlp.* entries of a reference model load with strict=True."""
    import hyena_dna_b200 as H
    with open(os.path.join(GOLD, "ref_model_keys.json")) as f:
        rec = json.load(f)
    D = rec["d_model"]
    prefix = "backbone.layers.0.mlp."
    want = {k[len(prefix):]: v["shape"] for k, v in rec["keys"].items() if k.startswith(prefix)}
    assert set(want) == {"fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias"}
    m = H.Mlp(D, hidden_features=want["fc1.weight"][0], activation=partial(F.gelu, approximate="tanh"))
    assert _shapes(m) == want
    m.load_state_dict({k: torch.randn(s) for k, s in want.items()}, strict=True)


def test_default_sizes():
    import hyena_dna_b200 as H
    m = H.Mlp(24)
    assert m.fc1.in_features == 24 and m.fc1.out_features == 96 and m.fc2.out_features == 24
    assert m.approximate == "none" and m.return_residual is False
    assert H.Mlp(8, activation=partial(F.gelu, approximate="tanh")).approximate == "tanh"
    assert H.Mlp(8, activation=partial(F.gelu, approximate="none")).approximate == "none"
    assert H.Mlp(8, activation=partial(F.gelu)).approximate == "none"


@pytest.mark.parametrize("activation", [F.relu, F.silu, torch.tanh, partial(F.gelu, approximate="sigmoid"),
                                        lambda x: F.gelu(x), partial(F.gelu, approximate="tanh", out=None),
                                        partial(F.relu, inplace=False)])
def test_unsupported_activation_raises(activation):
    import hyena_dna_b200 as H
    with pytest.raises(H.HyenaB200Error):
        H.Mlp(16, activation=activation)


def test_cpu_forward_raises():
    import hyena_dna_b200 as H
    for kw in ({}, {"return_residual": True}, {"bias1": False, "bias2": False}):
        m = H.Mlp(16, **kw)
        with pytest.raises(H.HyenaB200Error):
            m(torch.randn(2, 8, 16))


def test_fused_gelu_abi_rejects_bad_arguments():
    from importlib import import_module
    _lib = import_module("hyena_dna_b200._lib")
    L = _lib.lib()
    p = 256                          # never dereferenced: the argument checks come first
    err = lambda: L.hyena_b200_last_error().decode()
    assert L.hyena_b200_proj_gemm_gelu(p, p, 8, 0, None, 3, p, 1, 64, 8, 8, p, 1 << 20, None) != 0 and "activation" in err()
    assert L.hyena_b200_proj_gemm_gelu(p, p, 8, 0, None, 1, p, 1, 0, 8, 8, p, 1 << 20, None) != 0 and "bad shape" in err()
    assert L.hyena_b200_proj_gemm_dgelu(p, p, 8, 0, None, 1, p, 1, 64, 8, 8, p, 1 << 20, None) != 0 and "null" in err()
    assert L.hyena_b200_proj_gemm_dgelu(p, p, 8, 0, p, 2, p, 1, 64, 8, 8, p, 1 << 20, None) != 0 and "overlap" in err()
    assert L.hyena_b200_proj_wgrad_gelu(p, p, 0, p, 0, 0.0, 1, 64, 8, 8, p, 1 << 20, None) != 0 and "activation" in err()
    names = [L.hyena_b200_kind_name(i).decode() for i in range(L.hyena_b200_kind_count())]
    assert {"proj_gemm<gelu>", "proj_gemm<dgelu>", "proj_wgrad<gelu>"} <= set(names)


def test_fused_gelu_kernels_are_built_for_sm90a():
    from importlib import import_module
    _lib = import_module("hyena_dna_b200._lib")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump (CUDA toolkit) not available")
    out = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in subprocess.run([tool, "-lelf", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = set(re.findall(r"Function (\S+):", out))
    for fn in (1, 2):                # FN_GELU_TANH, FN_GELU_ERF
        assert f"_ZN2hy2pg16proj_gemm_kernelILi128ELi1ELi1ELi{fn}EEEvNS0_4ArgsE14CUtensorMap_st" in funcs   # GELU prologue
        assert f"_ZN2hy2pg16proj_gemm_kernelILi128ELi0ELi0ELi{fn}EEEvNS0_4ArgsE14CUtensorMap_st" in funcs   # dGELU epilogue
        assert f"_ZN2hy2wg12wgrad_kernelILi{fn}EEEvNS0_4ArgsE14CUtensorMap_stS3_" in funcs                  # GELU converter
