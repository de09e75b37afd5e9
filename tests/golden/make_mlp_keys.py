"""Record the state-dict keys and shapes of the UNMODIFIED reference block MLP (run in the build container only).

    python tests/golden/make_mlp_keys.py

Builds flash-attention/flash_attn/modules/mlp.py:Mlp (imported from /root/reference) for a few constructor settings --
the default hidden size, an explicit hidden / output size, and bias1 / bias2 switched off -- and writes
tests/golden/ref_mlp_keys.json: per case the constructor keywords and every state_dict key with its shape.
tests/test_mlp_cpu.py builds hyena_dna_b200.Mlp with the same keywords and compares.
"""
import json
import os
import sys

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
CASES = [
    {"in_features": 16},
    {"in_features": 32, "hidden_features": 64, "out_features": 24},
    {"in_features": 16, "bias1": False},
    {"in_features": 16, "bias2": False},
    {"in_features": 16, "hidden_features": 48, "bias1": False, "bias2": False},
]


def main():
    sys.path.insert(0, os.path.join(REF, "flash-attention"))
    from flash_attn.modules.mlp import Mlp
    assert os.path.realpath(sys.modules["flash_attn"].__file__).startswith(REF), "flash_attn did not resolve to the reference tree"
    rec = []
    for kw in CASES:
        sd = Mlp(**kw).state_dict()
        rec.append({"kwargs": kw, "keys": {k: list(v.shape) for k, v in sd.items()}})
    with open(os.path.join(OUT, "ref_mlp_keys.json"), "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    print(len(rec), "cases")


if __name__ == "__main__":
    main()
