"""Time the block MLP fwd+bwd: hyena_dna_b200.Mlp (fused-GELU wgmma kernels) against the reference composition in torch.

    python tools/bench_mlp.py [--B 1] [--L 1048576] [--D 256] [--H 1024] [--steps 20] [--warmup 3]

Both runs use the same input, upstream gradient and weights, fp32 with TF32 off, GELU approximate="tanh" (HyenaDNA's
create_mlp_cls).  The two variants alternate step by step in one process, each step timed with CUDA events.  Prints, per
variant, the median and mean ms per step, the fp32-equivalent rate (12 B L D H FLOP per fwd+bwd step: three GEMM pairs of
2 B L D H each way) and torch.cuda.max_memory_allocated over its steps (x, dy, weights and gradients included), then one
profiled step of the library variant by kernel class, and the card (read-only nvidia-smi query) it ran on.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from functools import partial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1)
    ap.add_argument("--L", type=int, default=1 << 20)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--H", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    B, L, D, Hd = args.B, args.L, args.D, args.H
    gen = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, L, D, device=dev, generator=gen).requires_grad_(True)
    dy = torch.randn(B, L, D, device=dev, generator=gen)
    ours = H.Mlp(D, hidden_features=Hd, activation=partial(F.gelu, approximate="tanh")).to(dev)
    W1, b1, W2, b2 = (p.detach().clone().requires_grad_(True) for p in
                      (ours.fc1.weight, ours.fc1.bias, ours.fc2.weight, ours.fc2.bias))
    if H.ops.proj_mode() != "tc":
        raise SystemExit(f"projection mode {H.ops.proj_mode()!r}: the fused kernels run in mode 'tc' only")

    def step_ours():
        y = ours(x)
        y.backward(dy)

    def step_torch():          # the reference Mlp.forward (flash_attn/modules/mlp.py:26-30) and its autograd
        y = F.linear(F.gelu(F.linear(x, W1, b1), approximate="tanh"), W2, b2)
        y.backward(dy)

    variants = {"hyena_dna_b200.Mlp": (step_ours, list(ours.parameters())), "torch": (step_torch, [W1, b1, W2, b2])}

    def clear(params):
        x.grad = None
        for p in params:
            p.grad = None

    for _ in range(args.warmup):
        for fn, params in variants.values():
            clear(params)
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    peak = {k: 0 for k in variants}
    for _ in range(args.steps):
        for name, (fn, params) in variants.items():
            clear(params)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
            peak[name] = max(peak[name], torch.cuda.max_memory_allocated(dev))

    flop = 12.0 * B * L * D * Hd
    res = {"shape": {"B": B, "L": L, "D": D, "H": Hd}, "steps": args.steps, "warmup": args.warmup, "fp32_equiv_flop": flop}
    for name in variants:
        med = statistics.median(ms[name])
        res[name] = {"ms_median": med, "ms_mean": statistics.fmean(ms[name]), "ms_min": min(ms[name]),
                     "ms_max": max(ms[name]), "tflops_fp32_equiv": flop / med / 1e9, "max_memory_allocated_gib": peak[name] / 2**30}
        print(f"{name:20s} {med:9.2f} ms/step (median; mean {res[name]['ms_mean']:.2f}, min {res[name]['ms_min']:.2f}, "
              f"max {res[name]['ms_max']:.2f})  {flop / med / 1e9:6.1f} TFLOP/s fp32-equivalent  "
              f"max_memory_allocated {peak[name] / 2**30:.2f} GiB")

    clear(variants["hyena_dna_b200.Mlp"][1])
    H._lib.profile_begin()
    step_ours()
    prof = H._lib.profile_end()
    res["profile_ms"] = {k: round(v[0], 3) for k, v in sorted(prof.items())}
    print("one profiled step of hyena_dna_b200.Mlp:", ", ".join(f"{k} {v[0]:.2f} ms ({v[1]})" for k, v in sorted(prof.items())))
    res["card"] = card()
    print("card:", res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
