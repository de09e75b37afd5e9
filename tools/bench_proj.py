"""Time the six projection calls of one HyenaOperator fwd+bwd step, one by one, on the wgmma kernels.

    python tools/bench_proj.py [--L 1048576] [--D 256] [--reps 20] [--warmup 3] [--rounds 3] [--libs A.so B.so ...]

B = 1, fp32, TF32 off.  The calls and their shapes are the ones bench.py's step issues (order 2, 3 D = 768 in_proj outputs):
in_proj fwd, out_proj fwd, out_proj dgrad, in_proj dgrad with the fused transposed short filter (FIR), out_proj wgrad and
in_proj wgrad with FIR.  Each call is warmed up, then timed `--reps` times with CUDA events around the single call.

With `--libs`, every library is run in its own subprocess (HYENA_B200_LIB), the libraries alternating round by round, so that
builds of the same ABI are compared in one command on one card.  Prints per library and call the median and spread (min, max)
in ms over all rounds, the rate in TF32 MMA TFLOP/s (3xTF32: three MMA products per fp32 multiply-add) and its fraction of
the data sheet's dense TF32 495 TFLOP/s, whether every library produced the same output bits, and the card (read-only
nvidia-smi query).
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATASHEET_TF32 = 495e12
CALLS = ["in_proj fwd", "out_proj fwd", "out_proj dgrad", "in_proj dgrad+FIR", "out_proj wgrad", "in_proj wgrad+FIR"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def mma_flop(L, D):
    """TF32 MMA FLOP per call: 2 L K N multiply-add FLOP, three MMA products each."""
    C = 3 * D
    kn = {"in_proj fwd": D * C, "out_proj fwd": D * D, "out_proj dgrad": D * D, "in_proj dgrad+FIR": C * D,
          "out_proj wgrad": D * D, "in_proj wgrad+FIR": C * D}
    return {k: 3 * 2.0 * L * v for k, v in kn.items()}


def worker(args):
    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_proj needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    L, D, C = args.L, args.D, 3 * args.D
    gen = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=gen)
    u, y_pre, dy, ds = rnd(1, L, D), rnd(1, D, L), rnd(1, L, D), rnd(1, C, L)
    W_in, W_out, b_out, taps = rnd(C, D) / D ** 0.5, rnd(D, D) / D ** 0.5, rnd(D), rnd(C, 3)
    ops = H.ops
    calls = {
        "in_proj fwd": lambda: ops.proj_gemm(u, 0, W_in, False, 0),
        "out_proj fwd": lambda: ops.proj_gemm(y_pre, 1, W_out, False, 1, bias=b_out),
        "out_proj dgrad": lambda: ops.proj_gemm(dy, 0, W_out, True, 0),
        "in_proj dgrad+FIR": lambda: ops.proj_gemm(ds, 1, W_in, True, 1, fir=taps),
        "out_proj wgrad": lambda: ops.proj_wgrad(y_pre, dy, transposed_out=True),
        "in_proj wgrad+FIR": lambda: ops.proj_wgrad(ds, u, fir=taps),
    }
    res = {}
    for name in CALLS:
        fn = calls[name]
        for _ in range(args.warmup):
            out = fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        digest = hashlib.sha256(out.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
        res[name] = {"ms": ms, "sha256": digest}
        del out
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--L", type=int, default=1 << 20)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--libs", nargs="*", default=None, help="library builds to compare (default: the in-tree build)")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)

    libs = args.libs or [""]
    ms = {lib: {c: [] for c in CALLS} for lib in libs}
    sha = {lib: {} for lib in libs}
    for _ in range(args.rounds):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["HYENA_B200_LIB"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--L", str(args.L), "--D", str(args.D),
                   "--reps", str(args.reps), "--warmup", str(args.warmup)]
            out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
            r = json.loads(out.strip().splitlines()[-1])
            for c in CALLS:
                ms[lib][c] += r[c]["ms"]
                sha[lib].setdefault(c, set()).add(r[c]["sha256"])

    flop = mma_flop(args.L, args.D)
    res = {"shape": {"B": 1, "L": args.L, "D": args.D}, "reps": args.reps, "warmup": args.warmup, "rounds": args.rounds,
           "libs": {}}
    for lib in libs:
        name = lib or "in-tree"
        res["libs"][name] = {}
        total = 0.0
        print(f"== {name}")
        for c in CALLS:
            med = statistics.median(ms[lib][c])
            total += med
            rate = flop[c] / med / 1e9
            res["libs"][name][c] = {"ms_median": med, "ms_min": min(ms[lib][c]), "ms_max": max(ms[lib][c]),
                                    "tflops_tf32_mma": rate, "frac_datasheet_tf32": rate * 1e12 / DATASHEET_TF32}
            print(f"  {c:18s} {med:8.3f} ms (min {min(ms[lib][c]):.3f}, max {max(ms[lib][c]):.3f})  "
                  f"{rate:6.1f} TFLOP/s TF32 MMA  {rate * 1e12 / DATASHEET_TF32:.3f} of 495")
        res["libs"][name]["total_ms"] = total
        print(f"  {'six calls':18s} {total:8.3f} ms")
    same = all(len(sha[lib][c]) == 1 for lib in libs for c in CALLS) and \
        all(sha[lib][c] == sha[libs[0]][c] for lib in libs for c in CALLS)
    res["outputs_bit_identical"] = same
    print("outputs bit-identical across rounds and libraries:", same)
    res["card"] = card()
    print("card:", res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
