"""Time incremental decoding (HyenaOperator.step / Backbone.step, csrc/decode.cuh) at long histories.

    python tools/bench_decode.py [--steps 50] [--warmup 5] [--layers 8] [--skip-backbone]

1. One order-2 operator, B = 1, D = 256, l_max = 2^20: per-step latency at history t in {2^10, 2^14, 2^17, 2^20 - 64}.
   The history is filled with random values and the cache's position set to t (a step's cost does not depend on the
   values); every timed step is the plain step at t, which reads the whole history.  Reports the median step time (CUDA events around op.step: in_proj / out_proj matrix-vector products and the
   library kernels), the median kernel time of the library launches (profiler window over the same steps) and the achieved
   bandwidth on the algorithmic bytes 4 D t + e B D t: the fp32 filter once plus the history of every batch row, e bytes
   per element (4 for fp32, 2 for a 16-bit history).  --history-dtype, --batch and --positions list the configurations,
   run one after another in the same process (defaults: fp32, B = 1, the positions above).
2. A Backbone of `--layers` blocks (HyenaOperator + Mlp, d_model 256, H = 1024): tokens/s stepping at t = 2^20 - 64, against
   one torch.no_grad() forward of the same backbone at L = 2^20 -- what each new position costs without a cache.  With
   --graph the steps replay a StepGraph instead (and the forward is skipped); one backbone per --history-dtype, B = 1.
3. torch.cuda.max_memory_allocated of each part and DecodeCache.nbytes, and the card (read-only nvidia-smi query).
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


def _fill(cache, t, gen):
    for c in (cache.layers or [cache]):
        c.h[..., :t].normal_(generator=gen)
        c.tail.normal_(generator=gen)
        c.t = t


def _time_steps(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--skip-backbone", action="store_true")
    ap.add_argument("--history-dtype", nargs="+", default=["float32"], choices=["float32", "float16", "bfloat16"])
    ap.add_argument("--batch", type=int, nargs="+", default=[1])
    ap.add_argument("--positions", type=int, nargs="+", default=None, help="history lengths t (default 2^10 .. 2^20 - margin)")
    ap.add_argument("--graph", action="store_true", help="step the backbone through a StepGraph")
    args = ap.parse_args()

    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    Lmax, D, B = 1 << 20, 256, 1
    margin = args.steps + args.warmup + 2
    res = {"steps": args.steps, "warmup": args.warmup, "operator": {}, "card": card()}

    # ---- 1. one operator
    op = H.HyenaOperator(D, Lmax, order=2, emb_dim=5).to(dev)

    def step(x, cache):
        """op.step on the plain route at the cache's position (every step reads the whole history; the windowed route,
        DESIGN.md section 4.11, would read a window of it), without advancing it."""
        return op._step_with(x, cache, H.ops.decode_step)
    positions = args.positions or [1 << 10, 1 << 14, 1 << 17, Lmax - margin]
    multi = len(args.history_dtype) > 1 or len(args.batch) > 1
    for hname in args.history_dtype:
        hd = getattr(torch, hname)
        for B in args.batch:
            torch.cuda.reset_peak_memory_stats(dev)
            cache = op.allocate_decode_cache(B, Lmax, history_dtype=hd)
            e = cache.h.element_size()
            out = res["operator"].setdefault(f"{hname}/B{B}", {}) if multi else res["operator"]
            res["operator_cache_nbytes" + (f"/{hname}/B{B}" if multi else "")] = cache.nbytes
            x = torch.randn(B, 1, D, device=dev, generator=gen)
            with torch.no_grad():
                for t in positions:
                    _fill(cache, t, gen)
                    ms = _time_steps(lambda: step(x, cache), args.steps, args.warmup)
                    _fill(cache, t, gen)
                    H._lib.profile_begin()
                    for _ in range(args.steps):
                        step(x, cache)
                    prof = H._lib.profile_end()
                    k_ms = prof["decode_step"][0] / args.steps
                    nbytes = 4.0 * D * t + e * B * D * t
                    med = statistics.median(ms)
                    out[str(t)] = {"step_ms_median": med, "step_ms_min": min(ms), "kernel_ms": k_ms,
                                   "algorithmic_bytes": nbytes, "gbps_kernel": nbytes / k_ms / 1e6,
                                   "gbps_step": nbytes / med / 1e6}
                    print(f"operator step {hname} B={B} t={t:8d}: {med:7.3f} ms/step (median; min {min(ms):.3f}), library "
                          f"kernels {k_ms:.3f} ms -> {nbytes / k_ms / 1e6:7.1f} GB/s kernel, {nbytes / med / 1e6:7.1f} GB/s "
                          "step")
            res["operator_max_memory_allocated_gib" + (f"/{hname}/B{B}" if multi else "")] = \
                torch.cuda.max_memory_allocated(dev) / 2**30
            del cache
            torch.cuda.empty_cache()
    del op
    torch.cuda.empty_cache()
    B = 1
    x = torch.randn(B, 1, D, device=dev, generator=gen)

    # ---- 2. backbone
    if not args.skip_backbone and args.graph:
        m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
        res["backbone_graph"] = {}
        for hname in args.history_dtype:
            torch.cuda.reset_peak_memory_stats(dev)
            cache = m.allocate_decode_cache(B, Lmax, history_dtype=getattr(torch, hname))
            _fill(cache, Lmax - margin, gen)
            with torch.no_grad():
                g = m.capture_step(cache, B)
                ms = _time_steps(lambda: g.step(x), args.steps, args.warmup)
            med = statistics.median(ms)
            res["backbone_graph"][hname] = {
                "layers": args.layers, "d_model": D, "t": Lmax - margin, "step_ms_median": med, "tokens_per_s": 1e3 / med,
                "cache_nbytes": cache.nbytes, "max_memory_allocated_gib": torch.cuda.max_memory_allocated(dev) / 2**30}
            print(f"backbone ({args.layers} layers + Mlp) StepGraph step, {hname} history, at t = {Lmax - margin}: "
                  f"{med:.3f} ms -> {1e3 / med:.1f} tokens/s; cache {cache.nbytes / 2**30:.2f} GiB")
            del g, cache
            torch.cuda.empty_cache()
    elif not args.skip_backbone:
        torch.cuda.reset_peak_memory_stats(dev)
        m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
        cache = m.allocate_decode_cache(B, Lmax)
        _fill(cache, Lmax - margin, gen)
        with torch.no_grad():
            ms = _time_steps(lambda: m.step(x, cache), args.steps, args.warmup)
        med = statistics.median(ms)
        peak_step = torch.cuda.max_memory_allocated(dev) / 2**30
        del cache
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        u = torch.randn(B, Lmax, D, device=dev, generator=gen)
        with torch.no_grad():
            fwd = _time_steps(lambda: m(u), 3, 1)
        fmed = statistics.median(fwd)
        res["backbone"] = {"layers": args.layers, "d_model": D, "mlp_hidden": 4 * D, "t": Lmax - margin,
                           "step_ms_median": med, "tokens_per_s": 1e3 / med, "cache_nbytes": H.DecodeCache.layout_nbytes(
                               B, D, 2, Lmax) * args.layers, "step_max_memory_allocated_gib": peak_step,
                           "forward_L_ms_median": fmed, "forward_max_memory_allocated_gib":
                           torch.cuda.max_memory_allocated(dev) / 2**30, "speedup_per_position": fmed / med}
        print(f"backbone ({args.layers} layers + Mlp) step at t = {Lmax - margin}: {med:.3f} ms -> {1e3 / med:.1f} tokens/s; "
              f"full no_grad forward at L = 2^20: {fmed:.1f} ms ({fmed / med:.0f}x a step)")
    print("card:", res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
