"""Time branched decode caches (DecodeCache.fork, DESIGN.md section 4.12) against cloning the cache per candidate.

    python tools/bench_fork.py [--layers 8] [--gen-steps 4096] [--skip-operator] [--skip-backbone] [--out FILE]

B = 1 context, D = 256, order 2, l_max = 2^20, fp32, TF32 off, CUDA events; the context's history is random (the cost does
not depend on its values).  For one operator and for a Backbone of --layers blocks with Mlp (H = 1024):
1. Candidate scoring at t0 in {2^17, 2^20 - 1024}: K in {4, 64, 256} candidates of n in {1, 64, 1000} positions.
     fork    cache.fork([0] * K, horizon) with the horizon the candidates need, then one extend of (K, n, D)
     clone   per candidate: a copy of the cache's state (history, tail, scratch; the filter shared) and extend (1, n, D);
             all K copies alive at once, as a caller scoring K candidates holds them.  Reported as "does not fit" when K
             copies do not fit in the free device memory.
2. Generation: K in {1, 16, 64} branches forked at 2^20 - --gen-steps, each stepped --gen-steps positions; aggregate
   positions per second, against one unbranched stream on the automatic route (windowed steps, section 4.11).
3. Route check (operator): both extend routes on branch histories of at most 4096 positions, at the end of the horizon.
4. Memory: nbytes of the branched caches and of one clone, the peak allocated while forking.
The card's name and power limit are read in the same run (read-only nvidia-smi query).
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


def _set_t(cache, t):
    for c in _caches(cache):
        c.t = t
        c.reset_window()


def _timed(fn, reps=3):
    """Median ms of fn() over reps calls, each synchronised, after one warm-up call -> (ms, last result)."""
    import torch
    out = fn()
    ms = []
    for _ in range(reps):
        del out
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), out


def _clone(cache):
    """What a caller without fork holds per candidate: the cache state copied, the filter shared."""
    import hyena_dna_b200 as H
    if cache.layers:
        return H.DecodeCache.stack(_clone(c) for c in cache.layers)
    c = H.DecodeCache(cache.owner, cache.batch_size, cache.max_seqlen, cache.lcap, cache.k, cache.bias, cache.h.clone(),
                      cache.tail.clone(), cache.s_t.clone(), cache.part.clone())
    c.t = cache.t
    return c


def _clone_bytes(cache):
    return sum(x.numel() * x.element_size() for c in _caches(cache) for x in (c.h, c.tail, c.s_t, c.part))


def _scoring(name, m, cache, D, gen, res):
    import torch
    rows = []
    for t0 in (1 << 17, (1 << 20) - 1024):
        for n in (1, 64, 1000):
            for K in (4, 64, 256):
                _set_t(cache, t0)
                u = torch.randn(K, n, D, device=gen.device, generator=gen)
                row = {"t0": t0, "n": n, "K": K}
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                fork_ms, br = _timed(lambda: cache.fork([0] * K, n + 4))
                row["fork_peak_extra_bytes"] = torch.cuda.max_memory_allocated() - base
                row["branched_nbytes"] = br.nbytes

                def ext():
                    _set_t(br, t0)
                    return m.extend(u, br)
                row["fork_ms"] = fork_ms
                row["branched_extend_ms"] = _timed(ext)[0]
                row["fork_total_ms"] = fork_ms + row["branched_extend_ms"]
                del br
                torch.cuda.empty_cache()
                need, free = K * _clone_bytes(cache), torch.cuda.mem_get_info()[0]
                row["clone_nbytes"] = _clone_bytes(cache)
                if need > free - (4 << 30):
                    row["clone_ms"] = "does not fit"
                else:
                    clones = []
                    try:
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for i in range(K):
                            clones.append(_clone(cache))
                            m.extend(u[i:i + 1], clones[-1])
                        e1.record()
                        e1.synchronize()
                        row["clone_ms"] = e0.elapsed_time(e1)
                    except torch.cuda.OutOfMemoryError:
                        row["clone_ms"] = "does not fit"
                    del clones
                    torch.cuda.empty_cache()
                rows.append(row)
                print(f"{name} scoring t0={t0} n={n} K={K}: fork {row['fork_ms']:.2f} ms + extend "
                      f"{row['branched_extend_ms']:.2f} ms; clone route {row['clone_ms']}", flush=True)
    res[name + "_scoring"] = rows


def _generation(name, m, cache, D, gen, steps, res):
    import torch
    t0 = (1 << 20) - steps
    out = {}
    for K in (1, 16, 64):
        _set_t(cache, t0)
        br = cache.fork([0] * K, steps)
        x = torch.randn(K, 1, D, device=gen.device, generator=gen)
        for _ in range(3):
            m.step(x, br)
        _set_t(br, t0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            m.step(x, br)
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        out[f"fork_K{K}"] = {"ms": ms, "positions_per_s": K * steps * 1e3 / ms, "nbytes": br.nbytes}
        print(f"{name} generation K={K}: {K * steps * 1e3 / ms:.0f} positions/s", flush=True)
        del br
        torch.cuda.empty_cache()
    x = torch.randn(1, 1, D, device=gen.device, generator=gen)
    _set_t(cache, t0)
    for _ in range(3):
        m.step(x, cache)
    _set_t(cache, t0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.step(x, cache)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1)
    out["single_stream_auto"] = {"ms": ms, "positions_per_s": steps * 1e3 / ms}
    print(f"{name} generation single stream (auto route): {steps * 1e3 / ms:.0f} positions/s", flush=True)
    res[name + "_generation"] = {"t0": t0, "steps": steps, **out}


def _routes(op, cache, D, gen, res):
    import torch
    import hyena_dna_b200 as H
    t0 = (1 << 20) - 4096
    rows = []
    for K in (1, 16):
        _set_t(cache, t0)
        br = cache.fork([0] * K, 4096)
        for n in (64, 256, 512, 1024, 2048):
            u = torch.randn(K, n, D, device=gen.device, generator=gen)
            row = {"K": K, "n": n, "j": 4096 - n}
            for route in ("direct", "fft"):
                def run():
                    br.t = t0 + 4096 - n
                    return op._extend(u, br, partial(H.ops.decode_branch_extend, fft=route == "fft"))
                row[route + "_ms"] = _timed(run)[0]
            rows.append(row)
            print(f"route check K={K} j={4096 - n} n={n}: direct {row['direct_ms']:.3f} ms, fft {row['fft_ms']:.3f} ms",
                  flush=True)
        del br
    res["operator_routes"] = rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--gen-steps", type=int, default=4096)
    ap.add_argument("--skip-operator", action="store_true")
    ap.add_argument("--skip-backbone", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_fork needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    Lmax, D = 1 << 20, 256
    res = {"card": card(), "B": 1, "D": D, "order": 2, "l_max": Lmax}
    print("card:", res["card"])
    with torch.no_grad():
        if not args.skip_operator:
            op = H.HyenaOperator(D, Lmax, order=2, emb_dim=5).to(dev)
            cache = op.allocate_decode_cache(1, Lmax)
            cache.h.normal_(generator=gen)
            cache.tail.normal_(generator=gen)
            _scoring("operator", op, cache, D, gen, res)
            _generation("operator", op, cache, D, gen, args.gen_steps, res)
            _routes(op, cache, D, gen, res)
            del cache, op
            torch.cuda.empty_cache()
        if not args.skip_backbone:
            m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                           mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
            cache = m.allocate_decode_cache(1, Lmax)
            for c in cache.layers:
                c.h.normal_(generator=gen)
                c.tail.normal_(generator=gen)
            res["backbone_layers"] = args.layers
            _scoring("backbone", m, cache, D, gen, res)
            _generation("backbone", m, cache, D, gen, args.gen_steps, res)
    print("card:", res["card"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
