"""Where the cycles of the projection GEMM kernel go: per-phase clock64() shares of the four proj_gemm calls of a step.

    make -C hyena-dna_b200/csrc EXTRA=-DHYENA_B200_PROJ_PHASES OBJDIR=build_phases OUT=../libhyena_b200_phases.so
    python tools/proj_phases.py --lib hyena-dna_b200/libhyena_b200_phases.so [--L 1048576] [--D 256] [--reps 5]

Needs a build with -DHYENA_B200_PROJ_PHASES: proj_gemm_kernel then adds, per warp, the cycles spent in each phase into a
device buffer (one row per CTA), read back through hyena_b200_proj_phases.  The calls and shapes are tools/bench_proj.py's:
B = 1, fp32, in_proj fwd, out_proj fwd, out_proj dgrad, in_proj dgrad with the fused transposed short filter (FIR).

Consumer phases, as a share of the consumer warps' cycles: waiting for a chunk's FULL barrier, loading and splitting the A
fragments (with the FIR / GELU prologue), MMA issue to wgmma_wait return, the chunk sum (and loop overhead), the epilogue.
Where the next chunk's fragments are loaded under this chunk's MMAs, that time counts as full_wait and prep, not mma.
Producer: its EMPTY waits as a share of its cycles.  Also printed: a CTA's cycles per K chunk, and the share of
those an MMA-bound schedule would need (12 m64n128k8 TF32 MMAs per warpgroup and chunk, two warpgroups on one SM's tensor
cores at 1024 TF32 multiply-adds per clock).  The counters perturb the schedule a little (clock reads, more registers), so
compare shares between builds with the flag, and take times from bench_proj.py.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PHASES = ["full_wait", "prep", "mma", "sum", "epilogue", "producer_empty_wait", "producer_issue"]
K_PHASES, PHASE_CTAS = 8, 1024
CALLS = ["in_proj fwd", "out_proj fwd", "out_proj dgrad", "in_proj dgrad+FIR"]
MMA_CYCLES_PER_CHUNK = 2 * 12 * 64 * 128 * 8 // 1024      # both warpgroups' MMAs of one chunk on one SM


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a -DHYENA_B200_PROJ_PHASES build of libhyena_b200.so")
    ap.add_argument("--L", type=int, default=1 << 20)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if args.lib:
        os.environ["HYENA_B200_LIB"] = os.path.abspath(args.lib)
    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("proj_phases needs a CUDA device")
    lib = H._lib.lib()
    if not hasattr(lib, "hyena_b200_proj_phases"):
        raise SystemExit("this library was built without -DHYENA_B200_PROJ_PHASES")
    read = lib.hyena_b200_proj_phases
    read.restype, read.argtypes = ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    buf = (ctypes.c_ulonglong * (PHASE_CTAS * K_PHASES))()

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    L, D, C = args.L, args.D, 3 * args.D
    gen = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=gen)
    u, y_pre, dy, ds = rnd(1, L, D), rnd(1, D, L), rnd(1, L, D), rnd(1, C, L)
    W_in, W_out, b_out, taps = rnd(C, D) / D ** 0.5, rnd(D, D) / D ** 0.5, rnd(D), rnd(C, 3)
    ops = H.ops
    calls = {
        "in_proj fwd": (lambda: ops.proj_gemm(u, 0, W_in, False, 0), D, C),
        "out_proj fwd": (lambda: ops.proj_gemm(y_pre, 1, W_out, False, 1, bias=b_out), D, D),
        "out_proj dgrad": (lambda: ops.proj_gemm(dy, 0, W_out, True, 0), D, D),
        "in_proj dgrad+FIR": (lambda: ops.proj_gemm(ds, 1, W_in, True, 1, fir=taps), C, D),
    }
    res = {"shape": {"B": 1, "L": L, "D": D}, "reps": args.reps, "calls": {}}
    for name in CALLS:
        fn, K, N = calls[name]
        fn()
        H._lib.check(read(None, 0, 1))
        for _ in range(args.reps):
            fn()
        H._lib.check(read(buf, PHASE_CTAS * K_PHASES, 1))
        tot = [sum(buf[c * K_PHASES + i] for c in range(PHASE_CTAS)) for i in range(K_PHASES)]
        cons = sum(tot[:5])
        prod = tot[5] + tot[6]
        chunks = args.reps * ((L + 127) // 128) * ((N + 127) // 128) * ((K + 31) // 32)
        per_chunk = cons / 8 / chunks                      # cycles of one CTA (eight consumer warps) per chunk
        r = {p: tot[i] / cons for i, p in enumerate(PHASES[:5])}
        r["producer_empty_wait"] = tot[5] / prod if prod else 0.0
        r["consumer_cycles_per_chunk"] = per_chunk
        r["mma_bound_share"] = MMA_CYCLES_PER_CHUNK / per_chunk
        res["calls"][name] = r
        print(f"{name:18s} " + "  ".join(f"{p} {r[p]:.3f}" for p in PHASES[:6]) +
              f"  cycles/chunk {per_chunk:.0f}  MMA-bound share {r['mma_bound_share']:.3f}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
