"""Time the two stages of the implicit filter's tensor-core backward on their own.

    python tools/bench_filter.py [--L 1048576] [--D 256] [--E 5] [--reps 20] [--warmup 3] [--rounds 3] [--libs A.so B.so ...]

The shapes are the ones bench.py's step runs (B = 1, D = 256, E = 5, L = 2^20).  Stage 1 (hyena_b200_filter_bwd_stage1)
turns dk into dh and the seven feature-major (64, L) arrays; stage 2 (hyena_b200_filter_bwd_stage2) reduces them over the
sequence into the filter's parameter gradients.  Each stage is warmed up, then timed `--reps` times with CUDA events around
the single call (stage 2's outputs are zeroed before the window).  The rate is over the compulsory HBM bytes (bench.py's
roofline counts the same): stage 1 reads dk and writes dh and the seven arrays, stage 2 reads dh and the seven arrays.
Also reported: whether stage 1's outputs are bit-identical across rounds and libraries, stage 2's error against an fp64
stage 2 on the same stage-1 arrays, and stage 2's time per kernel (torch.profiler, after the timed calls).

With `--libs`, every library is run in its own subprocess (HYENA_B200_LIB), the libraries alternating round by round, so that
builds of the same ABI are compared in one command on one card.  Prints per library and stage the median and spread (min,
max) in ms and GB/s, whether stage 2 returned the same bits on every call of a process, the largest difference between two
calls of a process and against the first library (both relative to each gradient's largest magnitude), and the card, power
limit and SM clock (read-only nvidia-smi query, taken after the timed calls).
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

STAGES = ["stage1", "stage2"]
GRADS = ["dW0", "db0", "dW1", "db1", "dW2", "db2", "dW3", "dfreq"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def hbm_bytes(L, D):
    arrays = 7 * 64 * 4.0 * L
    return {"stage1": 2 * 4.0 * D * L + arrays, "stage2": 4.0 * D * L + arrays}


def rel_diff(a, b):
    return float((a.double() - b.double()).abs().max() / a.double().abs().max().clamp_min(1e-300))


def worker(args):
    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_filter needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    L, D, E = args.L, args.D, args.E
    gen = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=gen)
    z, t = rnd(L, E), torch.linspace(0, 1, L, device=dev)
    W0, b0, W1, b1, W2, b2, W3 = rnd(64, E), rnd(64), rnd(64, 64) / 8, rnd(64), rnd(64, 64) / 8, rnd(64), rnd(D, 64) / 8
    freq, deltas = torch.ones(64, device=dev), rnd(D).abs()
    dk = rnd(D, L)
    dh, sc = torch.empty(D, L, device=dev), torch.empty(7, 64, L, device=dev)
    zT = z.t().contiguous()
    lib, st = H._lib.lib(), lambda: torch.cuda.current_stream().cuda_stream
    p = lambda x: x.data_ptr()
    grads = {"dW0": torch.zeros(64, E, device=dev), "db0": torch.zeros(64, device=dev),
             "dW1": torch.zeros(64, 64, device=dev), "db1": torch.zeros(64, device=dev),
             "dW2": torch.zeros(64, 64, device=dev), "db2": torch.zeros(64, device=dev),
             "dW3": torch.zeros(D, 64, device=dev), "dfreq": torch.zeros(64, device=dev)}

    def stage1():
        H._lib.check(lib.hyena_b200_filter_bwd_stage1(
            p(z), z.stride(0), p(t), p(W0), p(b0), p(W1), p(b1), p(W2), p(b2), p(W3), p(freq), p(deltas), 0.0, 1, L, E,
            64, D, p(dk), p(dh), p(sc), st()))

    def zero():
        for g in grads.values():
            g.zero_()

    def stage2():
        H._lib.check(lib.hyena_b200_filter_bwd_stage2(p(dh), p(sc), p(zT), *[p(grads[n]) for n in GRADS], L, E, D, st()))

    res, outs = {}, []
    for name, fn in (("stage1", stage1), ("stage2", stage2)):
        for _ in range(args.warmup):
            zero()
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            zero()                                   # outside the timed window: stage 2 adds into its outputs
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
            if name == "stage2" and len(outs) < 2:
                outs.append({n: g.clone() for n, g in grads.items()})
        res[name] = {"ms": ms}
        if name == "stage1":
            h = hashlib.sha256()
            for x in (dh, sc):
                h.update(x.cpu().numpy().tobytes())
            res["stage1_sha256"] = h.hexdigest()
    # stage 2 in fp64 on the same stage-1 arrays: the error of each build's gradients, relative to max |fp64|
    a1, a2, a3, dp1, dp2, dp3, X = sc.double().unbind(0)
    ref = {"dW0": dp1 @ zT.double().t(), "db0": dp1.sum(1), "dW1": dp2 @ a1.t(), "db1": dp2.sum(1), "dW2": dp3 @ a2.t(),
           "db2": dp3.sum(1), "dW3": dh.double() @ a3.t(), "dfreq": X.sum(1)}
    res["stage2_err_vs_fp64"] = {n: rel_diff(ref[n], outs[0][n]) for n in GRADS}
    del a1, a2, a3, dp1, dp2, dp3, X, ref
    # time per kernel of stage 2 (torch.profiler, after the timed calls)
    from torch.profiler import ProfilerActivity, profile
    zero()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            stage2()
        torch.cuda.synchronize()
    res["stage2_kernels_ms"] = {e.key[:60]: e.device_time_total / 5e3 for e in prof.key_averages() if e.device_time_total > 0}
    res["stage2_bit_identical"] = all(torch.equal(outs[0][n], outs[1][n]) for n in GRADS)
    res["stage2_run_to_run"] = {n: rel_diff(outs[0][n], outs[1][n]) for n in GRADS}
    torch.save({n: g.cpu() for n, g in outs[0].items()}, args.out)
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=1 << 20)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--E", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--libs", nargs="*", default=None, help="library builds to compare (default: the in-tree build)")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)

    import torch
    libs = args.libs or [""]
    ms = {lib: {s: [] for s in STAGES} for lib in libs}
    same = {lib: True for lib in libs}
    s1sha = {lib: set() for lib in libs}
    err64 = {lib: {n: 0.0 for n in GRADS} for lib in libs}
    kern = {lib: {} for lib in libs}
    spread = {lib: {n: 0.0 for n in GRADS} for lib in libs}
    vs_first = {lib: {n: 0.0 for n in GRADS} for lib in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            first = None
            for i, lib in enumerate(libs):
                env = dict(os.environ)
                if lib:
                    env["HYENA_B200_LIB"] = os.path.abspath(lib)
                out = os.path.join(tmp, f"{i}_{r}.pt")
                cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--L", str(args.L), "--D", str(args.D),
                       "--E", str(args.E), "--reps", str(args.reps), "--warmup", str(args.warmup), "--out", out]
                res = json.loads(subprocess.run(cmd, env=env, capture_output=True, text=True,
                                                check=True).stdout.strip().splitlines()[-1])
                for s in STAGES:
                    ms[lib][s] += res[s]["ms"]
                same[lib] &= res["stage2_bit_identical"]
                s1sha[lib].add(res["stage1_sha256"])
                for n in GRADS:
                    err64[lib][n] = max(err64[lib][n], res["stage2_err_vs_fp64"][n])
                kern[lib] = res["stage2_kernels_ms"]
                g = torch.load(out)
                first = first or g
                for n in GRADS:
                    spread[lib][n] = max(spread[lib][n], res["stage2_run_to_run"][n])
                    vs_first[lib][n] = max(vs_first[lib][n], rel_diff(first[n], g[n]))

    nbytes = hbm_bytes(args.L, args.D)
    summary = {"shape": {"B": 1, "L": args.L, "D": args.D, "E": args.E}, "reps": args.reps, "warmup": args.warmup,
               "rounds": args.rounds, "libs": {}}
    for lib in libs:
        name = lib or "in-tree"
        d = summary["libs"][name] = {}
        print(f"== {name}")
        for s in STAGES:
            med = statistics.median(ms[lib][s])
            d[s] = {"ms_median": med, "ms_min": min(ms[lib][s]), "ms_max": max(ms[lib][s]),
                    "gb_per_s": nbytes[s] / med / 1e6}
            print(f"  {s}  {med:8.3f} ms (min {min(ms[lib][s]):.3f}, max {max(ms[lib][s]):.3f})  "
                  f"{nbytes[s] / med / 1e6:7.0f} GB/s on {nbytes[s] / 1e9:.2f} GB")
        d["stage1+stage2_ms"] = d["stage1"]["ms_median"] + d["stage2"]["ms_median"]
        d["stage2_bit_identical_within_process"] = same[lib]
        d["stage2_run_to_run_rel"] = spread[lib]
        d["stage2_vs_first_lib_rel"] = vs_first[lib]
        print(f"  both stages {d['stage1+stage2_ms']:8.3f} ms; stage 2 bit-identical call to call: {same[lib]}")
        d["stage2_err_vs_fp64_rel"] = err64[lib]
        d["stage2_kernels_ms"] = kern[lib]
        d["stage1_sha256"] = sorted(s1sha[lib])
        print(f"  stage 2 call-to-call max rel diff: {max(spread[lib].values()):.2e}; vs first library: "
              f"{max(vs_first[lib].values()):.2e}")
        print("  stage 2 max error / max|fp64| per gradient: " + ", ".join(f"{n} {err64[lib][n]:.1e}" for n in GRADS))
        print("  stage 2 per kernel (ms, last round): " + ", ".join(f"{k} {v:.3f}" for k, v in kern[lib].items()))
    summary["stage1_outputs_bit_identical"] = len(set().union(*s1sha.values())) == 1
    print("stage 1 outputs (dh and the seven arrays) bit-identical across rounds and libraries:",
          summary["stage1_outputs_bit_identical"])
    summary["card"] = card()
    print("card:", summary["card"])
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
