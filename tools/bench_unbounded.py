"""Unbounded decode caches (max_seqlen=None, DESIGN.md section 4.20): generation and serving past the filter's l_max taps,
against a bounded cache that stops at its wall.  One JSON line per measurement.

  generate: an n_layer Backbone with Mlp, a prompt of l_max / 2 positions, then StepGraph steps.  Bounded: up to the wall
            (l_max - P tokens).  Unbounded: --gen-factor * l_max tokens (4 by default), sliding every S tokens.  Tokens/s,
            p50 / p99 / max of the synchronised per-token time, and the time of each slide (DecodeCache._make_room, timed
            between synchronisations).
  serve:    the continuous-batching trace of tools/bench_serve.py with total request lengths past l_max: B rows share one
            cache, finished rows are released and the next request admitted (left-padded), steps run under a StepGraph.
            Bounded: compact() when the position reaches Lcap, and a request stops at its row's wall (l_max - 4
            positions).  Unbounded: every request runs to its end.  Tokens/s and p50 / p99 request latency.
Inputs are random (no sampling).  The card's name and power limit are read in the same run.  Writes nothing but stdout.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_serve import card, now, pct  # noqa: E402


def backbone(D, n_layer, l_max, dev):
    import hyena_dna_b200 as H
    torch.manual_seed(0)
    m = H.Backbone(D, n_layer, partial(H.HyenaOperator, l_max=l_max, emb_dim=5, w=10.0),
                   mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True)
    return m.to(dev)


def generate(m, l_max, B, D, n, unbounded, dev):
    """-> (seconds, per-token times, slide times, tokens)."""
    import hyena_dna_b200 as H
    P = l_max // 2
    cache = m.allocate_decode_cache(B, None if unbounded else l_max)
    slides, make_room = [], H.DecodeCache._make_room

    def timed(self, k, step=False):
        if not self.unbounded:
            return 0
        a = now()
        r = make_room(self, k, step)
        if r:
            slides.append(now() - a)
        return r
    H.DecodeCache._make_room = timed
    try:
        with torch.no_grad():
            m.prefill(0.5 * torch.randn(B, P, D, device=dev), cache)
            graph = m.capture_step(cache, B)
            tok = 0.5 * torch.randn(B, 1, D, device=dev)
            n = n if unbounded else l_max - P
            times = []
            t0 = now()
            for _ in range(n):
                a = time.perf_counter()
                graph.step(tok)
                times.append(now() - a)
            total = now() - t0
    finally:
        H.DecodeCache._make_room = make_room
    return total, times, slides, n


def serve(m, trace, B, D, l_max, unbounded, dev):
    """-> (seconds, latencies, tokens generated, compactions)."""
    cache = m.allocate_decode_cache(B, None if unbounded else l_max)
    queue = list(range(len(trace)))
    left, lat, tokens, compactions = {}, [], 0, 0
    t0 = now()

    def admit(rows):
        reqs = [queue.pop(0) for _ in rows]
        lengths = [trace[i][0] for i in reqs]
        P = max(lengths)
        u = torch.zeros(len(rows), P, D, device=dev)
        for j, n in enumerate(lengths):
            u[j, P - n:] = 0.5 * torch.randn(n, D, device=dev)
        m.admit(u, cache, rows, lengths)
        for r, i in zip(rows, reqs):
            # bounded: the row stops 4 positions before its wall, so that compaction (a multiple of 4) always frees room
            left[r] = trace[i][1] if unbounded else min(trace[i][1], l_max - 4 - trace[i][0])
    with torch.no_grad():
        admit(list(range(min(B, len(queue)))))
        graph = m.capture_step(cache, B)
        tok = 0.5 * torch.randn(B, 1, D, device=dev)
        while left:
            if not unbounded and cache.t >= cache.lcap:
                compactions += 1
                assert cache.compact() > 0
            graph.step(tok)
            tokens += len(left)
            done = []
            for r in list(left):
                left[r] -= 1
                if left[r] <= 0:
                    done.append(r)
            if done:
                lat += [now() - t0] * len(done)
                for r in done:
                    del left[r]
                cache.release(done)
                rows = done[:len(queue)]
                if rows:
                    admit(rows)
    return now() - t0, lat, tokens, compactions


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--l-max", type=int, nargs="+", default=[1026, 1 << 17])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--gen-factor", type=float, default=4.0, help="unbounded generation: this many times l_max tokens")
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--serve-l-max", type=int, default=1026)
    ap.add_argument("--serve-batch", type=int, default=8)
    ap.add_argument("--requests", type=int, default=4, help="requests in the serving trace per batch row")
    ap.add_argument("--skip-generate", action="store_true")
    ap.add_argument("--skip-serve", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_unbounded needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    D = args.d_model
    if not args.skip_generate:
        for l_max in args.l_max:
            m = backbone(D, args.n_layer, l_max, dev)
            for B in args.batch:
                for unbounded in (False, True):
                    n = int(args.gen_factor * l_max)
                    total, times, slides, n = generate(m, l_max, B, D, n, unbounded, dev)
                    ms = [1e3 * x for x in times]
                    print(json.dumps({
                        "bench": "generate", "card": name, "power_limit": limit, "l_max": l_max, "batch": B,
                        "d_model": D, "n_layer": args.n_layer, "cache": "unbounded" if unbounded else "bounded",
                        "prompt": l_max // 2, "tokens": n, "tokens_per_s": round(B * n / total, 1),
                        "step_ms_p50": round(pct(ms, 0.5), 4), "step_ms_p99": round(pct(ms, 0.99), 4),
                        "step_ms_max": round(max(ms), 4), "slides": len(slides),
                        "slide_ms_mean": round(1e3 * sum(slides) / len(slides), 4) if slides else None}), flush=True)
            del m
            torch.cuda.empty_cache()
    if not args.skip_serve:
        l_max, B = args.serve_l_max, args.serve_batch
        rng = random.Random(0)
        trace = []
        for _ in range(args.requests * B):
            prompt = int(math.exp(rng.uniform(math.log(64), math.log(l_max))))
            trace.append((prompt, rng.randint(l_max // 2, 2 * l_max)))      # totals mostly past l_max
        m = backbone(D, args.n_layer, l_max, dev)
        serve(m, trace[:B], B, D, l_max, True, dev)                           # warm-up: module loading, captures
        for unbounded in (False, True):
            total, lat, tokens, compactions = serve(m, trace, B, D, l_max, unbounded, dev)
            print(json.dumps({
                "bench": "serve", "card": name, "power_limit": limit, "l_max": l_max, "batch": B, "d_model": D,
                "n_layer": args.n_layer, "cache": "unbounded" if unbounded else "bounded", "requests": len(trace),
                "past_l_max": sum(p + g > l_max for p, g in trace), "tokens": tokens,
                "tokens_per_s": round(tokens / total, 1), "latency_s_p50": round(pct(lat, 0.5), 3),
                "latency_s_p99": round(pct(lat, 0.99), 3), "compactions": compactions, "seconds": round(total, 3)}),
                flush=True)


if __name__ == "__main__":
    main()
