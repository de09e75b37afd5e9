"""Packed variable-length batches (forward(u, cu_seqlens=...), DESIGN.md section 4.18): one JSON line per configuration.

Each configuration runs one way of feeding the same sequences and reports real tokens/s and peak memory for a training
step (forward + backward) and a no-grad forward:
  packed  -- u (total, D) with cu_seqlens;
  mask    -- the batch left-padded to the longest sequence, forward(u, mask=...);
  loop    -- one call per sequence.
Models: one HyenaOperator and an n_layer Backbone with Mlp (D = 256).  Traces (seeded): 2048 sequences uniform in
[64, 1024], and the section 4.14 trace, 64 sequences log-uniform in [2^10, 2^17].  Median over --steps calls, host clock
around synchronised work; a separate profiled step gives the library's per-kind device times.  A configuration that runs
out of memory reports "oom".  The card's name and power limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import math
import os
import sys
import time
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_ragged import card  # noqa: E402


def trace(name):
    g = torch.Generator().manual_seed(0)
    if name == "uniform_64_1024":
        return torch.randint(64, 1025, (2048,), generator=g).tolist()
    lo, hi = math.log(1 << 10), math.log(1 << 17)
    return [int(math.exp(lo + (hi - lo) * float(x))) for x in torch.rand(64, generator=g)]


def make_calls(H, model, lengths, D, dev, how):
    """-> (list of (u, kwargs, dy) calls) feeding ``lengths`` the ``how`` way."""
    g = torch.Generator(device=dev).manual_seed(1)
    if how == "packed":
        total = sum(lengths)
        cu = torch.tensor([0] + list(torch.tensor(lengths).cumsum(0).tolist()), dtype=torch.int32, device=dev)
        u = 0.5 * torch.randn(total, D, device=dev, generator=g)
        return [(u, {"cu_seqlens": cu, "max_seqlen": max(lengths)}, torch.randn(total, D, device=dev, generator=g))]
    if how == "mask":
        P = max(lengths)
        mask = torch.arange(P, device=dev)[None, :] >= torch.tensor([P - n for n in lengths], device=dev)[:, None]
        u = 0.5 * torch.randn(len(lengths), P, D, device=dev, generator=g)
        dy = torch.randn(len(lengths), P, D, device=dev, generator=g) * mask[:, :, None]
        return [(u, {"mask": mask}, dy)]
    return [(0.5 * torch.randn(1, n, D, device=dev, generator=g), {}, torch.randn(1, n, D, device=dev, generator=g))
            for n in lengths]


def step(model, calls, train):
    for u, kw, dy in calls:
        if train:
            ud = u.detach().requires_grad_(True)
            model(ud, **kw).backward(dy)
        else:
            with torch.no_grad():
                model(u, **kw)


def measure(H, model, calls, train, steps, warmup):
    params = list(model.parameters())
    for _ in range(warmup):
        step(model, calls, train)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t = []
    for _ in range(steps):
        for p in params:
            p.grad = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step(model, calls, train)
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    peak = torch.cuda.max_memory_allocated() - base
    torch.cuda.synchronize()
    H._lib.profile_begin()
    step(model, calls, train)
    torch.cuda.synchronize()
    kinds = {k: round(v[0], 3) for k, v in sorted(H._lib.profile_end().items()) if v[1]}
    t.sort()
    return t[len(t) // 2], peak, kinds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--only", choices=["operator", "backbone"], default=None)
    ap.add_argument("--trace", choices=["uniform_64_1024", "loguniform_2e10_2e17"], default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_varlen needs a CUDA device"
    import hyena_dna_b200 as H
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    D = args.d_model
    for tr in ([args.trace] if args.trace else ["uniform_64_1024", "loguniform_2e10_2e17"]):
        lengths = trace(tr)
        P = max(lengths)
        for what in ([args.only] if args.only else ["operator", "backbone"]):
            torch.manual_seed(0)
            mixer = partial(H.HyenaOperator, l_max=P, emb_dim=5, w=10.0)
            model = (mixer(D) if what == "operator" else
                     H.Backbone(D, args.n_layer, mixer, mlp_cls=partial(H.Mlp, hidden_features=4 * D),
                                residual_in_fp32=True)).to(dev)
            for how in ("packed", "mask", "loop"):
                for train in (True, False):
                    rec = {"bench": "varlen", "gpu": name, "power_limit": limit, "trace": tr, "what": what, "D": D,
                           "n_layer": args.n_layer if what == "backbone" else 1, "sequences": len(lengths),
                           "real_tokens": sum(lengths), "longest": P, "how": how,
                           "step": "fwd+bwd" if train else "no_grad fwd", "steps": args.steps}
                    try:
                        calls = make_calls(H, model, lengths, D, dev, how)
                        sec, peak, kinds = measure(H, model, calls, train, args.steps, args.warmup)
                        rec.update(ms=round(1e3 * sec, 2), real_tokens_per_s=round(sum(lengths) / sec),
                                   peak_gib=round(peak / 2 ** 30, 2), kinds_ms=kinds)
                    except torch.cuda.OutOfMemoryError:
                        rec["result"] = "oom"
                    calls = None
                    for p in model.parameters():
                        p.grad = None
                    torch.cuda.empty_cache()
                    print(json.dumps(rec), flush=True)
            del model
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
