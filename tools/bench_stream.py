"""Streaming forward (forward(u, stream=True), DESIGN.md section 4.21): time and peak memory.  One JSON line per
measurement.

  operator: one HyenaOperator (order 2) at --D, for each l_max of --l-max over L = --L positions (B = 1): the window route
            at every window length of --windows (0: the plan's rule) against one window of the whole row (L_b = 2^20,
            when the row fits in one).  Median of --reps synchronised calls after a warm-up call.
  backbone: an --n-layer Backbone with Mlp at --D and --bb-l-max over each L of --bb-L: stream=True against an unbounded
            DecodeCache's prefill of l_max positions and extends of the rest (DecodeCache runs extends in pieces of
            min(4096, l_max) positions), and against hand-made overlapping chunks: --chunk positions of outputs per chunk,
            each chunk given n_layer (l_max - 1) positions of context and run through forward(stream=True), keeping its
            outputs.  One timed call each after a warm-up at a smaller L.
Inputs are random.  The card's name and power limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import os
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_serve import card, now  # noqa: E402


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.reset_peak_memory_stats()
        a = now()
        fn()
        ts.append(now() - a)
    return sorted(ts)[len(ts) // 2], torch.cuda.max_memory_allocated() / 2**30


def operator(args, dev, name, limit):
    import hyena_dna_b200 as H
    from hyena_dna_b200 import ops
    for l_max in args.l_max:
        torch.manual_seed(0)
        op = H.HyenaOperator(args.D, l_max, emb_dim=5, w=10.0).to(dev)
        u = torch.randn(1, args.L, args.D, device=dev)
        Lbs = [w or ops.stream_window_length(ops.stream_context(l_max, 2)) for w in args.windows]
        if args.L <= 1 << 20:
            Lbs.append(1 << 20)
        for L_b in dict.fromkeys(Lbs):
            if L_b <= l_max + 1:
                continue
            plan = ops.stream_plan(args.L, l_max, 2, 1, L_b=L_b)
            nwin = sum(len(plan.windows(e - s)) for s, a, e in plan.chunks)
            with torch.no_grad():
                op._forward_stream(u, plan)
                sec, gib = timed(lambda: op._forward_stream(u, plan), args.reps)
            print(json.dumps({"bench": "stream_operator", "D": args.D, "l_max": l_max, "L": args.L, "L_b": L_b,
                              "rule": L_b == ops.stream_window_length(ops.stream_context(l_max, 2)),
                              "windows": nwin, "ms": round(1e3 * sec, 3), "peak_gib": round(gib, 2), "gpu": name,
                              "power_limit": limit}), flush=True)
        del op, u
        torch.cuda.empty_cache()


def backbone(args, dev, name, limit):
    import hyena_dna_b200 as H
    torch.manual_seed(0)
    l_max = args.bb_l_max
    m = H.Backbone(args.D, args.n_layer, partial(H.HyenaOperator, l_max=l_max, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=4 * args.D), residual_in_fp32=True).to(dev)
    ctx = args.n_layer * (l_max - 1)

    def stream(u):
        return m(u, stream=True)

    def decode(u):
        c = m.allocate_decode_cache(u.shape[0], None)
        return torch.cat([m.prefill(u[:, :l_max], c), m.extend(u[:, l_max:], c)], dim=1)

    def chunks(u):
        L = u.shape[1]
        out = torch.empty_like(u)
        for a in range(0, L, args.chunk):
            e = min(L, a + args.chunk)
            s = max(0, a - ctx)
            out[:, a:e] = m(u[:, s:e], stream=True)[:, a - s:]
        return out

    with torch.no_grad():
        w = torch.randn(1, 3 * l_max + 5, args.D, device=dev)
        for fn in (stream, decode, chunks):
            fn(w)
        for L in args.bb_L:
            u = torch.randn(1, L, args.D, device=dev)
            for what, fn in (("stream", stream), ("decode", decode), ("chunks", chunks)):
                if what == "decode" and L > args.decode_max:
                    continue
                sec, gib = timed(lambda: fn(u), 1)
                print(json.dumps({"bench": "stream_backbone", "route": what, "n_layer": args.n_layer, "D": args.D,
                                  "l_max": l_max, "L": L, "chunk": args.chunk if what == "chunks" else None,
                                  "s": round(sec, 3), "positions_per_s": round(L / sec), "peak_gib": round(gib, 2),
                                  "gpu": name, "power_limit": limit}), flush=True)
            del u
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", choices=["operator", "backbone", "all"], default="all")
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--L", type=int, default=1 << 20)
    ap.add_argument("--l-max", type=int, nargs="+", default=[1026, 32770])
    ap.add_argument("--windows", type=int, nargs="+", default=[0, 4096, 8192, 16384, 65536, 262144])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--bb-l-max", type=int, default=1026)
    ap.add_argument("--bb-L", type=int, nargs="+", default=[1 << 20, 1 << 22])
    ap.add_argument("--chunk", type=int, default=1 << 16)
    ap.add_argument("--decode-max", type=int, default=1 << 22)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_stream needs a CUDA device")
    dev = torch.device("cuda:0")
    name, limit = card()
    if args.what in ("operator", "all"):
        operator(args, dev, name, limit)
    if args.what in ("backbone", "all"):
        backbone(args, dev, name, limit)


if __name__ == "__main__":
    main()
