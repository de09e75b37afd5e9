"""Packed prompts into a decode cache (prefill / admit with cu_seqlens, DESIGN.md section 4.19): one JSON line per
measurement.  Model: an n_layer Backbone with Mlp, D = 256.

  (a) prefill: the section 4.14 traces (8 prompts log-uniform in [2^10, 2^17]; 64 prompts log-uniform in [2^10, 2^14]),
      fed packed (Backbone.prefill with cu_seqlens), left-padded to the longest (lengths=) and as one one-row prefill per
      prompt.  Median over --steps calls, host clock around synchronised work, peak memory above the model; a separate
      profiled call gives the library's per-kind device times.  Out of memory is reported as "oom".
  (b) serving: tools/bench_serve.py's continuous batching trace (B rows, --requests per row, prompts log-uniform up to
      --serve-max-len), admitting left-padded prompts and packed prompts, same trace: tokens/s, p50/p99 latency, or "oom".
  (c) the Mlp on a row count that is not a multiple of 4 (the packed layout, total = 3 mod 4): fc1 + fc2 as MlpFn on the
      row count itself against Mlp, which rounds it up to a multiple of 4 under no_grad, alternated, CUDA events.
The card's name and power limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import math
import os
import random
import sys
import time
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_serve import card, continuous, pct  # noqa: E402


def trace(B, hi, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo, hi = math.log(1 << 10), math.log(hi)
    return [int(math.exp(lo + (hi - lo) * float(x))) for x in torch.rand(B, generator=g)]


def prefill_calls(m, lengths, D, dev, how):
    """-> a function running one prefill of ``lengths`` the ``how`` way into fresh caches."""
    g = torch.Generator(device=dev).manual_seed(1)
    P = max(lengths)
    if how == "packed":
        u = 0.5 * torch.randn(sum(lengths), D, device=dev, generator=g)
        cu = torch.tensor([0] + torch.tensor(lengths).cumsum(0).tolist(), dtype=torch.int32)
        return lambda: m.prefill(u, m.allocate_decode_cache(len(lengths), P), cu_seqlens=cu)
    if how == "padded":
        u = 0.5 * torch.randn(len(lengths), P, D, device=dev, generator=g)
        return lambda: m.prefill(u, m.allocate_decode_cache(len(lengths), P), lengths=lengths)
    us = [0.5 * torch.randn(1, n, D, device=dev, generator=g) for n in lengths]
    return lambda: [m.prefill(u, m.allocate_decode_cache(1, u.shape[1])) for u in us]


def measure(H, run, steps, warmup):
    with torch.no_grad():
        for _ in range(warmup):
            run()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t = []
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run()
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
        peak = torch.cuda.max_memory_allocated() - base
        H._lib.profile_begin()
        run()
        torch.cuda.synchronize()
        kinds = {k: round(v[0], 3) for k, v in sorted(H._lib.profile_end().items()) if v[1]}
    t.sort()
    return t[len(t) // 2], peak, kinds


def backbone(H, D, n_layer, l_max, dev):
    torch.manual_seed(0)
    return H.Backbone(D, n_layer, partial(H.HyenaOperator, l_max=l_max, emb_dim=5, w=10.0),
                      mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)


def part_a(H, args, dev, name, limit):
    D = args.d_model
    for B, hi in ((8, 1 << 17), (64, 1 << 14)):
        lengths = trace(B, hi)
        m = backbone(H, D, args.n_layer, max(lengths), dev)
        for how in ("packed", "padded", "separate"):
            rec = {"bench": "packed_prefill", "gpu": name, "power_limit": limit, "B": B, "longest": max(lengths),
                   "real_tokens": sum(lengths), "D": D, "n_layer": args.n_layer, "how": how, "steps": args.steps}
            try:
                sec, peak, kinds = measure(H, prefill_calls(m, lengths, D, dev, how), args.steps, args.warmup)
                rec.update(ms=round(1e3 * sec, 2), peak_gib=round(peak / 2 ** 30, 2), kinds_ms=kinds)
            except torch.cuda.OutOfMemoryError:
                rec["result"] = "oom"
            torch.cuda.empty_cache()
            print(json.dumps(rec), flush=True)
        del m
        torch.cuda.empty_cache()


def part_b(H, args, dev, name, limit):
    D, B, max_len = args.d_model, args.serve_batch, args.serve_max_len
    rng = random.Random(0)
    tr = [(int(round(math.exp(rng.uniform(math.log(1 << 10), math.log(max_len))))), rng.randint(64, 1024))
          for _ in range(args.requests * B)]
    lcap = max_len + 2 * 1024
    gen = sum(n for _, n in tr)
    for hname in args.history_dtype:
        for packed in (False, True):
            rec = {"bench": "packed_serve", "gpu": name, "power_limit": limit, "B": B, "max_len": max_len, "D": D,
                   "n_layer": args.n_layer, "requests": len(tr), "generated": gen, "history_dtype": hname,
                   "admit": "packed" if packed else "left-padded"}
            m = backbone(H, D, args.n_layer, lcap, dev)
            try:
                with torch.no_grad():
                    m.prefill(0.5 * torch.randn(2, 1024, D, device=dev), m.allocate_decode_cache(2, 2048))
                    torch.cuda.empty_cache()
                    torch.cuda.reset_peak_memory_stats()
                    sec, lat, adm, _ = continuous(m, tr, B, D, lcap, dev, getattr(torch, hname), packed=packed)
                rec.update(tokens_per_s=round(gen / sec, 1), seconds=round(sec, 2), latency_p50_s=round(pct(lat, 0.5), 3),
                           latency_p99_s=round(pct(lat, 0.99), 3), admit_ms_mean=round(1e3 * sum(adm) / len(adm), 2),
                           peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
            except torch.cuda.OutOfMemoryError:
                rec["result"] = "oom"
            del m
            torch.cuda.empty_cache()
            print(json.dumps(rec), flush=True)


def part_c(H, args, dev, name, limit):
    D = args.d_model
    torch.manual_seed(0)
    mlp = H.Mlp(D, hidden_features=4 * D).to(dev)
    for total in (sum(trace(8, 1 << 17)) // 4 * 4 + 3, 2048 * 544 + 3):
        x = 0.5 * torch.randn(1, total, D, device=dev)
        runs = {"unrounded": lambda: H.ops.MlpFn.apply(x, mlp.fc1.weight, mlp.fc1.bias, mlp.fc2.weight, mlp.fc2.bias,
                                                       mlp.approximate),
                "rounded": lambda: mlp(x)}
        ms = {k: [] for k in runs}
        with torch.no_grad():
            same = torch.equal(runs["unrounded"](), runs["rounded"]())
            for _ in range(args.steps + 1):
                for k, f in runs.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    f()
                    e.record()
                    torch.cuda.synchronize()
                    ms[k].append(s.elapsed_time(e))
            kinds = {}
            for k, f in runs.items():
                H._lib.profile_begin()
                f()
                torch.cuda.synchronize()
                kinds[k] = {kk: round(v[0], 3) for kk, v in sorted(H._lib.profile_end().items()) if v[1]}
        rec = {"bench": "mlp_rows", "gpu": name, "power_limit": limit, "rows": total, "D": D, "H": 4 * D,
               "bit_identical": same, "kinds_ms": kinds}
        for k in runs:
            v = sorted(ms[k][1:])
            rec[f"{k}_ms"] = round(v[len(v) // 2], 3)
        print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", nargs="+", default=["c", "a", "b"], choices=["a", "b", "c"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--serve-batch", type=int, default=64)
    ap.add_argument("--serve-max-len", type=int, default=1 << 17)
    ap.add_argument("--requests", type=int, default=2, help="requests in the serving trace per batch row")
    ap.add_argument("--history-dtype", nargs="+", default=["float32"], choices=["float32", "float16", "bfloat16"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_packed_prefill needs a CUDA device"
    import hyena_dna_b200 as H
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    for part in args.part:
        {"a": part_a, "b": part_b, "c": part_c}[part](H, args, dev, name, limit)


if __name__ == "__main__":
    main()
