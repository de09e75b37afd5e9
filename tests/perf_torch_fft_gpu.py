"""Comparator measurement (not a pytest test): the reference's own GPU path -- the same torch ops the
reference HyenaOperator executes (restated in oracle/hyena_oracle.py), i.e. cuBLAS + cuDNN + cuFFT via
torch.fft -- timed on cuda:0 next to this repo's operator.  This is the ">= 10x" denominator of
BASELINE.json's north_star at L = 1,048,576 (the reference's csrc/fftconv extension cannot run past
L = 8192).  Run on a GPU machine; prints one JSON line.

    python tests/perf_torch_fft_gpu.py [--seqlen L] [--d-model D] [--batch B] [--steps K]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import hyena_oracle as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqlen", type=int, default=1 << 20)
    ap.add_argument("--d-model", type=int, default=256)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--tf32", action="store_true")
    a = ap.parse_args()
    import hyena_dna_b200 as H
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = a.tf32
    torch.backends.cudnn.allow_tf32 = a.tf32
    B, L, D = a.batch, a.seqlen, a.d_model
    g = torch.Generator().manual_seed(0)
    P = O.init_params(D, L, emb_dim=5, w=10.0, generator=g, init_std=0.02)
    u, _ = O.nucleotide_activations(B, L, D)
    dy = torch.randn(B, L, D, generator=g)
    Pd = {k: v.to(dev) for k, v in P.items()}
    ud, dyd = u.to(dev), dy.to(dev)

    def ref_step():
        return O.operator_fwd_bwd(ud, Pd, dyd)

    sd = dict(P)
    for extra in ("filter_fn.implicit_filter.3.freq", "filter_fn.implicit_filter.5.freq"):
        sd[extra] = sd["filter_fn.implicit_filter.1.freq"]
    op = H.HyenaOperator(D, L, emb_dim=5, w=10.0, lr_pos_emb=0.0)
    op.load_state_dict(sd)
    op = op.to(dev)
    ug = ud.clone().requires_grad_(True)

    def our_step():
        for p in op.parameters():
            p.grad = None
        ug.grad = None
        y = op(ug)
        y.backward(dyd)
        return y

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.steps

    ms_ref = timeit(ref_step)
    torch.cuda.empty_cache()
    ms_our = timeit(our_step)
    y_ref, du_ref, _ = ref_step()
    y = our_step()
    err = float((y - y_ref).abs().max()); sc = float(y_ref.abs().max())
    print(json.dumps({"shape": {"B": B, "L": L, "D": D}, "tf32": a.tf32,
                      "torch_fft_gpu_ms": ms_ref, "hyena_b200_ms": ms_our, "speedup": ms_ref / ms_our,
                      "torch_fft_gpu_nt_s": B * L / ms_ref * 1e3, "hyena_b200_nt_s": B * L / ms_our * 1e3,
                      "max_abs_diff_y": err, "max_abs_y": sc}))


if __name__ == "__main__":
    main()
