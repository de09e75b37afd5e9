"""Serving a request trace with a fixed number of batch rows (DESIGN.md section 4.15): one JSON line per configuration.

  (a) continuous batching: the rows share one cache; when a request finishes its row is released and the next request
      is admitted into it (Backbone.admit), generation runs under one StepGraph, and the cache is compacted when the
      position reaches Lcap;
  (b) static batching: B requests at a time, one left-padded prefill (Backbone.prefill with lengths), then B-row
      generation under a StepGraph until the longest of the B finishes.
Every request of the seeded trace is queued at the start; its latency is the time from the start of the run to its last
token.  Prompt lengths are log-uniform in [min_len, max_len], generation lengths uniform in [gen_min, gen_max]; the inputs
are random (no sampling).  Also times decode_shift alone and gives its rate on 8 (O-1) B D t bytes.  Times are wall-clock
around synchronised work; the card's name and power limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import math
import os
import random
import subprocess
import sys
import time
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:          # the numbers are still reported; the card is then named by torch only
        return torch.cuda.get_device_name(0), "unknown"


def now():
    torch.cuda.synchronize()
    return time.perf_counter()


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(math.ceil(q * len(xs))) - 1)]


def continuous(m, trace, B, D, lcap, dev, hd=torch.float32, packed=False):
    """(a): -> (seconds, latencies, admit times, compact times, compactions).  ``packed``: each admission's prompts are
    packed back to back (Backbone.admit with cu_seqlens) instead of left-padded to the longest."""
    cache = m.allocate_decode_cache(B, lcap, history_dtype=hd)
    queue = list(range(len(trace)))
    left, lat, adm, cmp_ = {}, [], [], []
    t0 = now()

    def admit(rows):
        reqs = [queue.pop(0) for _ in rows]
        P = max(trace[i][0] for i in reqs)
        lengths = [trace[i][0] for i in reqs]
        if packed:
            u = 0.5 * torch.randn(sum(lengths), D, device=dev)
            cu = torch.tensor([0] + torch.tensor(lengths).cumsum(0).tolist(), dtype=torch.int32)
        else:
            u = torch.zeros(len(rows), P, D, device=dev)
            for j, i in enumerate(reqs):
                u[j, P - lengths[j]:] = 0.5 * torch.randn(lengths[j], D, device=dev)
        a = now()
        if packed:
            m.admit(u, cache, rows, cu_seqlens=cu)
        else:
            m.admit(u, cache, rows, lengths)
        adm.append(now() - a)
        for r, i in zip(rows, reqs):
            left[r] = [i, trace[i][1]]
    with torch.no_grad():
        admit(list(range(min(B, len(queue)))))
        graph = m.capture_step(cache, B)
        tok = 0.5 * torch.randn(B, 1, D, device=dev)
        while left:
            if cache.t >= lcap:
                a = now()
                assert cache.compact() > 0, "no room: Lcap must exceed the longest request by gen_max"
                cmp_.append(now() - a)
            graph.step(tok)
            done = []
            for r in list(left):
                left[r][1] -= 1
                if left[r][1] == 0:
                    done.append(r)
            if done:
                tnow = now() - t0
                lat += [tnow] * len(done)
                for r in done:
                    del left[r]
                cache.release(done)
                rows = done[:len(queue)]
                if rows:
                    P = max(trace[i][0] for i in queue[:len(rows)])
                    g = max([left[r][1] for r in left] + [trace[i][1] for i in queue[:len(rows)]])
                    if max(cache.t, P) + g > lcap:
                        a = now()
                        cache.compact()
                        cmp_.append(now() - a)
                    admit(rows)
    return now() - t0, lat, adm, cmp_


def static(m, trace, B, D, dev, hd=torch.float32):
    """(b): -> (seconds, latencies, prefill times)."""
    lat, pre = [], []
    t0 = now()
    with torch.no_grad():
        for g0 in range(0, len(trace), B):
            group = trace[g0:g0 + B]
            k = len(group)
            lengths = [p for p, _ in group]
            P, G = max(lengths), max(n for _, n in group)
            u = torch.zeros(k, P, D, device=dev)
            for j, n in enumerate(lengths):
                u[j, P - n:] = 0.5 * torch.randn(n, D, device=dev)
            cache = m.allocate_decode_cache(k, P + G, history_dtype=hd)
            a = now()
            m.prefill(u, cache, lengths=lengths)
            pre.append(now() - a)
            graph = m.capture_step(cache, k)
            tok = 0.5 * torch.randn(k, 1, D, device=dev)
            ends = sorted(n for _, n in group)
            for i in range(1, G + 1):
                graph.step(tok)
                while ends and ends[0] == i:
                    lat.append(now() - t0)
                    ends.pop(0)
            del graph, cache
    return now() - t0, lat, pre


def shift_rate(m, B, D, lcap, dev, reps=5, hd=torch.float32):
    """hyena_b200_decode_shift (or its _h16 twin) on one layer's cache at t = lcap - 8, left by 4096 and back, alternated:
    (ms per shift, GB/s on 2 e (O-1) B D t bytes, the read and the write of every history word below t, e bytes each)."""
    import hyena_dna_b200 as H
    c = m.layers[0].mixer.allocate_decode_cache(B, lcap, history_dtype=hd)
    fn, t, stream = H.ops._decode_fn("shift", c.h), lcap - 8, torch.cuda.current_stream().cuda_stream

    def shift(pos, by):
        H._lib.check(fn(c.h.data_ptr(), B, D, c.order, pos, by, lcap, stream))
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shift(t, -4096)
    shift(t - 4096, 4096)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        shift(t, -4096)
        shift(t - 4096, 4096)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / (2 * reps)
    nbytes = 2 * c.h.element_size() * (c.order - 1) * B * D * t
    del c
    return ms, nbytes / ms / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 64])
    # a 64-row cache of 2^17 positions takes 69 GB over 8 layers: B = 64 stops at 2^14
    ap.add_argument("--max-len", type=int, nargs="+", default=[1 << 17, 1 << 14],
                    help="longest prompt, one per --batch entry")
    ap.add_argument("--min-len", type=int, default=1 << 10)
    ap.add_argument("--gen-min", type=int, default=64)
    ap.add_argument("--gen-max", type=int, default=1024)
    ap.add_argument("--requests", type=int, default=3, help="requests in the trace per batch row")
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--history-dtype", nargs="+", default=["float32"], choices=["float32", "float16", "bfloat16"],
                    help="the decode caches' history dtype (DESIGN.md section 4.16); several: each in turn, same trace")
    ap.add_argument("--skip-static", action="store_true", help="run continuous batching (a) only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_serve needs a CUDA device"
    import hyena_dna_b200 as H
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    D = args.d_model
    for (B, max_len), hname in [(bm, h) for bm in zip(args.batch, args.max_len) for h in args.history_dtype]:
        hd = getattr(torch, hname)
        rng = random.Random(args.seed)
        trace = [(int(round(math.exp(rng.uniform(math.log(args.min_len), math.log(max_len))))),
                  rng.randint(args.gen_min, args.gen_max)) for _ in range(args.requests * B)]
        # the shared clock: after a compaction the position is the longest live request, which may still generate
        # gen_max tokens while a new one is admitted and generates gen_max more
        lcap = max_len + 2 * args.gen_max
        torch.manual_seed(0)
        m = H.Backbone(D, args.n_layer, partial(H.HyenaOperator, l_max=lcap, emb_dim=5, w=10.0),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
        gen = sum(n for _, n in trace)
        rec = {"bench": "serve", "gpu": name, "power_limit": limit, "B": B, "D": D, "n_layer": args.n_layer,
               "requests": len(trace), "prompt_sum": sum(p for p, _ in trace), "generated": gen, "lcap": lcap,
               "history_dtype": hname, "cache_nbytes": args.n_layer * H.DecodeCache.layout_nbytes(B, D, 2, lcap, hd)}
        with torch.no_grad():
            w = min(B, 2)                    # warm-up of the library's set-up at this model's shapes
            m.prefill(0.5 * torch.randn(w, 1024, D, device=dev), m.allocate_decode_cache(w, 2048))
            torch.cuda.empty_cache()
            sec, lat, adm, cmp_ = continuous(m, trace, B, D, lcap, dev, hd)
            rec.update(a_tokens_per_s=gen / sec, a_seconds=sec, a_latency_p50_s=pct(lat, 0.5), a_latency_p99_s=pct(lat, 0.99),
                       a_admits=len(adm), a_admit_ms_mean=1e3 * sum(adm) / len(adm), a_admit_ms_max=1e3 * max(adm),
                       a_compactions=len(cmp_), a_compact_ms_mean=1e3 * sum(cmp_) / len(cmp_) if cmp_ else None,
                       a_compact_ms_max=1e3 * max(cmp_) if cmp_ else None)
            torch.cuda.empty_cache()
            if not args.skip_static:
                sec, lat, pre = static(m, trace, B, D, dev, hd)
                rec.update(b_tokens_per_s=gen / sec, b_seconds=sec, b_latency_p50_s=pct(lat, 0.5),
                           b_latency_p99_s=pct(lat, 0.99), b_prefills=len(pre), b_prefill_ms_mean=1e3 * sum(pre) / len(pre))
            torch.cuda.empty_cache()
            ms, gbs = shift_rate(m, B, D, lcap, dev, hd=hd)
            rec.update(shift_ms=ms, shift_t=lcap - 8, shift_gb_per_s=gbs)
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in rec.items()}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
