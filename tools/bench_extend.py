"""Time extending a decode cache by n positions at once (HyenaOperator.extend, csrc/decode_extend.cuh) and find where
the direct Toeplitz kernel stops beating the FFT route.

    python tools/bench_extend.py [--reps 5] [--warmup 2] [--layers 8] [--skip-backbone] [--out FILE]

1. One order-2 operator, B = 1, D = 256, l_max = 2^20, history t in {2^14, 2^17, 2^20 - n}, n in {1, 4, 16, 64, 256,
   1024, 8192}.  The history is filled with random values and the cache's position set to t before every call (the
   cost does not depend on the values).  Per (t, n), with CUDA events after warm-up, median of --reps:
     - extend(n) on each route (ops.decode_extend_direct / ops.decode_extend_fft) and on the route the library selects;
     - n successive step calls (one window, measured once);
     - one no_grad forward over t + n positions.
   Per route, the library kernels' time from the profiler (a separate window) and the rates on algorithmic work:
     direct kernel  bytes 4 D (t + n) (B + 1) (history and filter once), FMAs B D (n t + n (n + 1) / 2);
     FFT route      the whole history convolution (no FLOP count: reported as time only).
2. A Backbone of --layers blocks (HyenaOperator + Mlp, d_model 256, H = 1024) at t = 2^20 - 1000: scoring a 1000-position
   continuation by one extend against 1000 steps -> positions/s.
3. The card's name and power limit (read-only nvidia-smi query), in the same run.
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

TS = (1 << 14, 1 << 17, None)          # None: 2^20 - n
NS = (1, 4, 16, 64, 256, 1024, 8192)


def _fill(cache, t, gen):
    for c in (cache.layers or [cache]):
        c.h[..., :t].normal_(generator=gen)
        c.tail.normal_(generator=gen)
        c.t = t


def _set_t(cache, t):
    for c in (cache.layers or [cache]):
        c.t = t


def _time(fn, reps, warmup, reset):
    import torch
    for _ in range(warmup):
        reset()
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def _kernel_ms(fn, reset, reps):
    """Device time of the library's decode_extend_* launches (and of the FFT route's convolution kernels) per call."""
    import hyena_dna_b200 as H
    H._lib.profile_begin()
    for _ in range(reps):
        reset()
        fn()
    prof = H._lib.profile_end()
    skip = ("proj_gemm", "proj_prep")
    return {k: v[0] / reps for k, v in prof.items() if k not in skip}, {k: v[0] / reps for k, v in prof.items() if k in skip}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--skip-backbone", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_extend needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    Lmax, D, B = 1 << 20, 256, 1
    res = {"reps": args.reps, "warmup": args.warmup, "card": card(), "operator": [], "fft_min_n": H.ops.EXTEND_FFT_MIN_N}
    print("card:", res["card"])

    op = H.HyenaOperator(D, Lmax, order=2, emb_dim=5).to(dev)
    cache = op.allocate_decode_cache(B, Lmax)
    routes = {"direct": H.ops.decode_extend_direct, "fft": H.ops.decode_extend_fft}
    with torch.no_grad():
        for t0 in TS:
            for n in NS:
                t = Lmax - n if t0 is None else t0
                u = torch.randn(B, n, D, device=dev, generator=gen)
                _fill(cache, t, gen)
                reset = partial(_set_t, cache, t)
                row = {"t": t, "n": n, "selected": "fft" if H.ops.decode_extend_uses_fft(t, n) else "direct"}
                for name, core in routes.items():
                    fn = partial(op._extend, u, cache, core)
                    ms = _time(fn, args.reps, args.warmup, reset)
                    kms, pms = _kernel_ms(fn, reset, args.reps)
                    r = {"ms_median": statistics.median(ms), "ms_min": min(ms), "kernel_ms": kms, "proj_ms": pms}
                    if name == "direct":
                        k = kms.get("decode_extend_dot", float("nan"))
                        nbytes = 4.0 * D * (t + n) * (B + 1)
                        fma = B * D * (n * t + n * (n + 1) / 2)
                        r.update(dot_bytes=nbytes, dot_fma=fma, dot_gbps=nbytes / k / 1e6, dot_tflops=2 * fma / k / 1e9)
                    row[name] = r
                ms = _time(partial(op.extend, u, cache), args.reps, args.warmup, reset)
                row["extend_ms_median"] = statistics.median(ms)
                # n successive steps, one window after a warm-up step
                x1 = u[:, :1].contiguous()
                reset()
                op.step(x1, cache)
                reset()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for j in range(n):
                    op.step(u[:, j:j + 1], cache)
                e1.record()
                e1.synchronize()
                row["steps_ms"] = e0.elapsed_time(e1)
                del u
                uf = torch.randn(B, t + n, D, device=dev, generator=gen)
                ms = _time(lambda: op(uf), max(1, args.reps // 2), 1, lambda: None)
                row["forward_ms_median"] = statistics.median(ms)
                del uf
                row["speedup_vs_steps"] = row["steps_ms"] / row["extend_ms_median"]
                row["speedup_vs_forward"] = row["forward_ms_median"] / row["extend_ms_median"]
                res["operator"].append(row)
                d, f = row["direct"], row["fft"]
                print(f"t={t:8d} n={n:5d}: direct {d['ms_median']:9.3f} ms (dot {d['kernel_ms'].get('decode_extend_dot', 0):8.3f}"
                      f" ms, {d['dot_gbps']:7.1f} GB/s, {d['dot_tflops']:6.2f} TFLOP/s)  fft {f['ms_median']:9.3f} ms  "
                      f"selected={row['selected']:6s} extend {row['extend_ms_median']:9.3f} ms  {n} steps "
                      f"{row['steps_ms']:9.3f} ms  forward(t+n) {row['forward_ms_median']:8.2f} ms", flush=True)
    del cache, op
    torch.cuda.empty_cache()

    if not args.skip_backbone:
        N = 1000
        t = Lmax - N
        m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
        cache = m.allocate_decode_cache(B, Lmax)
        _fill(cache, t, gen)
        reset = partial(_set_t, cache, t)
        x = torch.randn(B, N, D, device=dev, generator=gen)
        with torch.no_grad():
            ms = _time(lambda: m.extend(x, cache), args.reps, args.warmup, reset)
            reset()
            m.step(x[:, :1], cache)
            reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for j in range(N):
                m.step(x[:, j:j + 1], cache)
            e1.record()
            e1.synchronize()
            steps_ms = e0.elapsed_time(e1)
        med = statistics.median(ms)
        res["backbone"] = {"layers": args.layers, "d_model": D, "mlp_hidden": 4 * D, "t": t, "n": N,
                           "selected": "fft" if H.ops.decode_extend_uses_fft(t, N) else "direct",
                           "extend_ms_median": med, "positions_per_s_extend": N * 1e3 / med, "steps_ms": steps_ms,
                           "positions_per_s_steps": N * 1e3 / steps_ms}
        print(f"backbone ({args.layers} layers + Mlp) at t = {t}: 1000-position continuation by extend {med:.1f} ms "
              f"-> {N * 1e3 / med:.0f} positions/s; by 1000 steps {steps_ms:.1f} ms -> {N * 1e3 / steps_ms:.0f} positions/s")
    print("card:", res["card"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
