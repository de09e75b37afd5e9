"""Training steps on left-padded batches (forward(u, mask=...), DESIGN.md section 4.17): one JSON line per configuration.

  operator (fwd + bwd of one HyenaOperator, order 2, D = 256):
    B = 1, P = 2^20 with an all-ones mask against the plain step (what the masking itself costs);
    B = 8, P = 2^17 with lengths log-uniform in [2^10, 2^17], masked against the same batch unmasked (the reference's
    semantics: the pads flow into every convolution);
  backbone (fwd + bwd of an n_layer Backbone with Mlp, D = 256) at (B = 64, P = 2^12) and (B = 8, P = 2^15), masked with
  log-uniform lengths against the same batch unmasked.
The variants are alternated step by step after a warm-up of each; median and range over --steps steps, CUDA events around
synchronised work.  A separate profiled step of each variant gives the library's per-kind device times (the masked modes
count under the kinds of the plain ones).  The card's name and power limit are read in the same run.  Writes nothing but
stdout.
"""
import argparse
import json
import math
import os
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_ragged import card, timed  # noqa: E402


def log_uniform(B, lo, hi):
    """B lengths from hi down to lo, log-uniformly spaced (the longest is hi)."""
    return [int(round(math.exp(math.log(hi) - (math.log(hi) - math.log(lo)) * i / max(B - 1, 1)))) for i in range(B)]


def left_mask(lengths, P, dev):
    return torch.arange(P, device=dev)[None, :] >= torch.tensor([P - n for n in lengths], device=dev)[:, None]


def run(model, u, dy, params, mask):
    for p in params:
        p.grad = None
    ud = u.detach().requires_grad_(True)
    y = model(ud, mask=mask) if mask is not None else model(ud)
    y.backward(dy)


def measure(H, rec, model, u, dy, variants, steps, warmup):
    params = list(model.parameters())
    for _ in range(warmup):
        for _, mask in variants:
            run(model, u, dy, params, mask)
    times = {name: [] for name, _ in variants}
    for _ in range(steps):                               # alternated: the variants see the same machine state
        for name, mask in variants:
            times[name].append(timed(lambda: run(model, u, dy, params, mask)))
    for name, t in times.items():
        t.sort()
        rec[f"{name}_ms"] = t[len(t) // 2]
        rec[f"{name}_range"] = [t[0], t[-1]]
    for name, mask in variants:                          # per-kind device times, profiled apart from the timed steps
        torch.cuda.synchronize()
        H._lib.profile_begin()
        run(model, u, dy, params, mask)
        torch.cuda.synchronize()
        rec[f"{name}_kinds_ms"] = {k: round(v[0], 3) for k, v in sorted(H._lib.profile_end().items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--only", choices=["operator", "backbone"], default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ragged_train needs a CUDA device"
    import hyena_dna_b200 as H
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    D = args.d_model
    cases = []
    if args.only in (None, "operator"):
        cases += [("operator", 1, 1 << 20, "all-ones"), ("operator", 8, 1 << 17, "log-uniform")]
    if args.only in (None, "backbone"):
        cases += [("backbone", 64, 1 << 12, "log-uniform"), ("backbone", 8, 1 << 15, "log-uniform")]
    for what, B, P, how in cases:
        torch.manual_seed(0)
        if what == "operator":
            model = H.HyenaOperator(D, P, emb_dim=5, w=10.0).to(dev)
        else:
            model = H.Backbone(D, args.n_layer, partial(H.HyenaOperator, l_max=P, emb_dim=5, w=10.0),
                               mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
        lengths = [P] * B if how == "all-ones" else log_uniform(B, min(1 << 10, P), P)
        u = 0.5 * torch.randn(B, P, D, device=dev)
        dy = torch.randn(B, P, D, device=dev) * left_mask(lengths, P, dev)[:, :, None]
        rec = {"bench": "ragged_train", "what": what, "gpu": name, "power_limit": limit, "B": B, "P": P, "D": D,
               "n_layer": args.n_layer if what == "backbone" else 1, "mask": how, "lengths_sum": sum(lengths),
               "steps": args.steps}
        measure(H, rec, model, u, dy, [("masked", left_mask(lengths, P, dev)), ("plain", None)], args.steps,
                args.warmup)
        print(json.dumps({k: (round(v, 3) if isinstance(v, float) else
                              [round(x, 3) for x in v] if isinstance(v, list) else v) for k, v in rec.items()}),
              flush=True)
        del model, u, dy
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
