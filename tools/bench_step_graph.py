"""Time generation with eager ``step`` against a CUDA-graph step (decode.StepGraph, DESIGN.md section 4.13).

    python tools/bench_step_graph.py [--layers 8] [--steps 4160] [--branch-steps 256] [--branches 64] [--repeats 2]
                                     [--out FILE]

1. One order-2 operator and a Backbone of --layers blocks with Mlp (B = 1, D = 256, hidden 1024, l_max = 2^20) at history
   t in {2^17, 2^20 - margin}.  The history is random (a step's cost does not depend on the values).  Before each run the
   cache is set back to t with no window and a full step count, so eager step and the graph both open a window at the
   first step and pay one refresh per WINDOW positions.  CUDA events around every step call (no synchronisation between
   steps) give the mean, p99 and max step time, and the mean time per position from the first event to the last.  Eager
   and graph runs alternate --repeats times; the run with the lower mean of each is reported.
2. --branches branches forked (horizon WINDOW) from one context of 2^20 - WINDOW positions, stepped --branch-steps
   positions from the fork, eager against the graph.
3. The card's name, power limit and SM clock (read-only nvidia-smi query) before and after the runs.
"""
import argparse
import json
import os
import statistics
import sys
from functools import partial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_mlp import card  # noqa: E402


def _caches(cache):
    return cache.layers or [cache]


def _timed(step, x, n):
    import torch
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for e0, e1 in ev:
        e0.record()
        step(x)
        e1.record()
    torch.cuda.synchronize()
    ms = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
    mean = ev[0][0].elapsed_time(ev[-1][1]) / n
    return {"n": n, "mean_ms_per_position": mean, "tokens_per_s": 1e3 / mean, "median_ms": statistics.median(ms),
            "p99_ms": ms[min(n - 1, int(0.99 * n))], "max_ms": ms[-1]}


def _compare(name, m, cache, reset, x, n, repeats, warmup=8):
    """Eager m.step against StepGraph.step for n positions after reset(), alternating; the lower-mean run of each."""
    import torch
    import hyena_dna_b200 as H
    reset()
    graph = H.StepGraph(m, cache, x.shape[0], x.dtype)
    runs = {"eager": [], "graph": []}
    for r in range(repeats):
        for how in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
            step = partial(m.step, cache=cache) if how == "eager" else graph.step
            reset()
            for _ in range(warmup):
                step(x)
            torch.cuda.synchronize()
            reset()
            runs[how].append(_timed(step, x, n))
    row = {how: min(rs, key=lambda s: s["mean_ms_per_position"]) for how, rs in runs.items()}
    row["speedup"] = row["eager"]["mean_ms_per_position"] / row["graph"]["mean_ms_per_position"]
    e, g = row["eager"], row["graph"]
    print(f"{name}: eager {e['tokens_per_s']:.0f} tok/s (mean {e['mean_ms_per_position']:.4f} ms, p99 {e['p99_ms']:.3f}, max "
          f"{e['max_ms']:.2f})  graph {g['tokens_per_s']:.0f} tok/s (mean {g['mean_ms_per_position']:.4f} ms, p99 "
          f"{g['p99_ms']:.3f}, max {g['max_ms']:.2f})  x{row['speedup']:.2f}", flush=True)
    return row


def _reset_to(ops, cache, t):
    def reset():
        for c in _caches(cache):
            c.t = t
            c.reset_window()
            c.steps = ops.WINDOW_AFTER_STEPS
    return reset


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--steps", type=int, default=4160)
    ap.add_argument("--branch-steps", type=int, default=256)
    ap.add_argument("--branches", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_step_graph needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    ops = H.ops
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    Lmax, D, B, W = 1 << 20, 256, 1, ops.WINDOW
    ts = (1 << 17, Lmax - args.steps - 64)
    res = {"card": card(), "steps": args.steps, "repeats": args.repeats, "window": W}
    print("card:", res["card"])
    x = torch.randn(B, 1, D, device=dev, generator=gen)

    with torch.no_grad():
        op = H.HyenaOperator(D, Lmax, order=2, emb_dim=5).to(dev)
        m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
        for name, mod in (("operator", op), ("backbone", m)):
            cache = mod.allocate_decode_cache(B, Lmax)
            for c in _caches(cache):
                c.h.normal_(generator=gen)
                c.tail.normal_(generator=gen)
            res[name] = [dict(t=t, **_compare(f"{name} t={t}", mod, cache, _reset_to(ops, cache, t), x, args.steps,
                                              args.repeats)) for t in ts]
            t0 = Lmax - W
            for c in _caches(cache):
                c.t = t0
                c.reset_window()
            br = cache.fork([0] * args.branches, W)
            xb = torch.randn(args.branches, 1, D, device=dev, generator=gen)

            def reset_branch(br=br):
                for c in _caches(br):
                    c.t = t0
            res[name + "_branches"] = dict(t0=t0, branches=args.branches, **_compare(
                f"{name} {args.branches} branches after t0={t0}", mod, br, reset_branch, xb, args.branch_steps, args.repeats))
            del cache, br
            torch.cuda.empty_cache()
    res["backbone_layers"] = args.layers
    res["card_after"] = card()
    print("card after the runs:", res["card_after"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
