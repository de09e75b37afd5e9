"""Batched generation from prompts of different lengths (DESIGN.md section 4.14): one JSON line per configuration.

  (a) ragged: one left-padded prefill of all B prompts (Backbone.prefill with lengths), then B-row generation under a
      StepGraph;
  (b) separate: B caches of one row each, each prompt prefilled unpadded, each cache stepped by its own StepGraph;
  (c) masked vs plain: Backbone.forward at the same (B, P) with and without lengths, alternated, to show what the masking
      costs.
Prompt lengths are spread log-uniformly over [min_len, max_len] (the longest is max_len); the model is a Backbone of
n_layer HyenaOperator blocks with Mlp.  Times are CUDA-event times around synchronised work; the card's name and power
limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import math
import os
import subprocess
import sys
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


def timed(fn, reps=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 64])
    # a 64-row cache of 2^17 positions takes 69 GB over 8 layers: B = 64 stops at 2^14
    ap.add_argument("--max-len", type=int, nargs="+", default=[1 << 17, 1 << 14],
                    help="longest prompt, one per --batch entry")
    ap.add_argument("--min-len", type=int, default=1 << 10)
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--n-layer", type=int, default=8)
    ap.add_argument("--new-tokens", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5, help="alternated repetitions of the forward pair in (c)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ragged needs a CUDA device"
    import hyena_dna_b200 as H
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    name, limit = card()
    D, N = args.d_model, args.new_tokens
    for B, max_len in zip(args.batch, args.max_len):
        torch.manual_seed(0)
        lmax = max_len + N
        m = H.Backbone(D, args.n_layer, partial(H.HyenaOperator, l_max=lmax, emb_dim=5, w=10.0),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D), residual_in_fp32=True).to(dev)
        lengths = [max_len] + [int(round(math.exp(math.log(args.min_len) + (math.log(max_len) - math.log(args.min_len))
                                                   * i / max(B - 1, 1)))) for i in range(B - 1)]
        P = max_len
        u = 0.5 * torch.randn(B, P, D, device=dev)
        tok = 0.5 * torch.randn(B, N, D, device=dev)
        rec = {"bench": "ragged", "gpu": name, "power_limit": limit, "B": B, "P": P, "D": D, "n_layer": args.n_layer,
               "new_tokens": N, "lengths_min": min(lengths), "lengths_sum": sum(lengths)}
        with torch.no_grad():
            # (a) one ragged prefill + B-row StepGraph generation
            m.prefill(u, m.allocate_decode_cache(B, lmax), lengths=lengths)           # warm-up of every prefill shape
            torch.cuda.empty_cache()
            cache = m.allocate_decode_cache(B, lmax)
            rec["a_prefill_ms"] = timed(lambda: m.prefill(u, cache, lengths=lengths))
            g = m.capture_step(cache, B)
            g.step(tok[:, :1])
            rec["a_step_ms"] = timed(lambda: [g.step(tok[:, i:i + 1]) for i in range(1, N)]) / (N - 1)
            del g, cache
            torch.cuda.empty_cache()
            # (b) B caches of one row each
            pre, stp = 0.0, 0.0
            for b, n in enumerate(lengths):
                c = m.allocate_decode_cache(1, lmax)
                pre += timed(lambda: m.prefill(u[b:b + 1, P - n:].contiguous(), c))
                gb = m.capture_step(c, 1)
                gb.step(tok[b:b + 1, :1])
                stp += timed(lambda: [gb.step(tok[b:b + 1, i:i + 1]) for i in range(1, N)]) / (N - 1)
                del gb, c
                torch.cuda.empty_cache()
            rec["b_prefill_ms"], rec["b_step_ms"] = pre, stp
            # (c) masked vs plain forward at the same (B, P), alternated after one warm-up of each
            m(u, lengths=lengths)
            m(u)
            tm, tp = [], []
            for _ in range(args.reps):
                tm.append(timed(lambda: m(u, lengths=lengths)))
                tp.append(timed(lambda: m(u)))
            tm.sort()
            tp.sort()
            rec.update(c_masked_ms=tm[len(tm) // 2], c_plain_ms=tp[len(tp) // 2], c_masked_range=[tm[0], tm[-1]],
                       c_plain_range=[tp[0], tp[-1]])
        print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in rec.items()}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
