"""Time generation (one position per step) on a long cache: the plain O(t) step against the windowed step with its FFT
refresh (HyenaOperator.step, ops.decode_window_plan, DESIGN.md section 4.11).

    python tools/bench_generate.py [--layers 8] [--windows 3] [--plain-steps 400] [--repeats 1] [--skip-operator]
                                   [--skip-backbone] [--out FILE]

1. One order-2 operator and a Backbone of --layers blocks with Mlp (B = 1, D = 256, H = 1024, l_max = 2^20), history
   t in {2^14, 2^17, 2^20 - margin} (and 2^15, 2^16 for the operator).  The history is random (a step's cost does not
   depend on the values); before each route the cache is set back to t with no window and no step count.  Routes:
     plain     WINDOW_MIN_T above every t: the parent's step
     windowed  WINDOW_MIN_T = WINDOW_AFTER_STEPS = 0: a window from the first step on
     auto      the shipped constants
   Per route, after warm-up steps: CUDA events around every step (no synchronisation between steps), giving the median,
   p99 and max step time, and the mean time per generated position from the first event to the last over --windows
   windows plus WINDOW_AFTER_STEPS steps (the refreshes included).  The plain route of the backbone runs --plain-steps
   positions (its per-step cost is flat over a few thousand positions).  With --repeats the routes run that many rounds
   in alternating order and the round with the median mean (the lower one of two) is reported.  The refresh on its own:
   median of 5 ops.decode_window_refresh calls at the same t (all layers for the backbone).
2. The interleaved workload "extend 64, step 1" at 2^20 - margin on the operator, plain and auto: mean time per position and
   the number of refreshes the automatic route paid.
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


def _caches(cache):
    return cache.layers or [cache]


def _reset(cache, t):
    for c in _caches(cache):
        c.t = t
        c.reset_window()


def _routes(ops):
    shipped = (ops.WINDOW_MIN_T, ops.WINDOW_AFTER_STEPS)
    return {"plain": (1 << 30, shipped[1]), "windowed": (0, 0), "auto": shipped}


def _set_route(ops, consts):
    ops.WINDOW_MIN_T, ops.WINDOW_AFTER_STEPS = consts


def _gen(step, x, n, warmup, reset):
    """n steps after `warmup` ones (each run from reset()) -> per-step ms list and the mean ms per position."""
    import torch
    reset()
    for _ in range(warmup):
        step(x)
    torch.cuda.synchronize()
    reset()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for e0, e1 in ev:
        e0.record()
        step(x)
        e1.record()
    torch.cuda.synchronize()
    ms = [e0.elapsed_time(e1) for e0, e1 in ev]
    return ms, ev[0][0].elapsed_time(ev[-1][1]) / n


def _stats(ms, mean):
    s = sorted(ms)
    return {"n": len(ms), "median_ms": statistics.median(s), "p99_ms": s[min(len(s) - 1, int(0.99 * len(s)))],
            "max_ms": s[-1], "mean_ms_per_position": mean}


def _refresh_ms(ops, cache, t, reps=5):
    import torch
    out = []
    for _ in range(reps):
        _reset(cache, t)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for c in _caches(cache):
            ops.decode_window_refresh(c)
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def _model(ops, name, m, cache, ts, x, args, res):
    rows = []
    routes = _routes(ops)
    shipped = routes["auto"]
    n_win = args.windows * ops.WINDOW + ops.WINDOW_AFTER_STEPS + 8
    for t in ts:
        row = {"t": t}
        # --repeats rounds, the route order reversed every other round (a long GPU-bound run before a host-bound one
        # changes what the latter measures); per route the round with the (lower) median mean is kept
        runs = {route: [] for route in routes}
        for r in range(args.repeats):
            for route in (list(routes) if r % 2 == 0 else list(routes)[::-1]):
                _set_route(ops, routes[route])
                n = min(n_win, args.plain_steps) if (route == "plain" and name == "backbone") else n_win
                ms, mean = _gen(partial(m.step, cache=cache), x, n, args.warmup, partial(_reset, cache, t))
                runs[route].append(_stats(ms, mean))
        for route, st in runs.items():
            st.sort(key=lambda s: s["mean_ms_per_position"])
            row[route] = dict(st[(len(st) - 1) // 2], means_of_rounds=[s["mean_ms_per_position"] for s in st])
        _set_route(ops, shipped)
        row["refresh_ms"] = _refresh_ms(ops, cache, t)
        row["refresh_in_plain_steps"] = row["refresh_ms"] / row["plain"]["median_ms"]
        if name == "backbone":
            for route in routes:
                row[route]["tokens_per_s"] = 1e3 / row[route]["mean_ms_per_position"]
        rows.append(row)
        p, w, a = row["plain"], row["windowed"], row["auto"]
        print(f"{name} t={t:8d}: plain {p['median_ms']:.3f} ms (mean {p['mean_ms_per_position']:.3f})  windowed median "
              f"{w['median_ms']:.3f} p99 {w['p99_ms']:.3f} max {w['max_ms']:.2f} mean {w['mean_ms_per_position']:.3f}  auto "
              f"mean {a['mean_ms_per_position']:.3f} max {a['max_ms']:.2f}  refresh {row['refresh_ms']:.2f} ms "
              f"= {row['refresh_in_plain_steps']:.1f} plain steps", flush=True)
    res[name] = rows


def _operator(ops, args, res, ts, t_inter, x, gen):
    """Section 1 for one operator, then section 2 (the interleaved workload)."""
    import torch
    import hyena_dna_b200 as H
    B, D = x.shape[0], x.shape[-1]
    op = H.HyenaOperator(D, 1 << 20, order=2, emb_dim=5).to(x.device)
    cache = op.allocate_decode_cache(B, 1 << 20)
    cache.h.normal_(generator=gen)
    cache.tail.normal_(generator=gen)
    with torch.no_grad():
        _model(ops, "operator", op, cache, ts, x, args, res)
        u = torch.randn(B, 64, D, device=x.device, generator=gen)
        refreshes = []
        real_refresh = ops.decode_window_refresh

        def counting_refresh(c):
            refreshes.append(c.t)
            real_refresh(c)
        ops.decode_window_refresh = counting_refresh
        inter = {}
        try:
            for route in ("plain", "auto"):
                _set_route(ops, _routes(ops)[route])
                for warm in (True, False):
                    _reset(cache, t_inter)
                    refreshes.clear()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(2 if warm else args.cycles):
                        op.extend(u, cache)
                        op.step(x, cache)
                    e1.record()
                    e1.synchronize()
                inter[route] = {"mean_ms_per_position": e0.elapsed_time(e1) / (65 * args.cycles),
                                "refreshes": len(refreshes)}
        finally:
            ops.decode_window_refresh = real_refresh
            _set_route(ops, _routes(ops)["auto"])
    res["interleaved"] = {"t": t_inter, "cycles": args.cycles, **inter}
    print(f"interleaved extend 64 + step 1 at t={t_inter}: plain {inter['plain']['mean_ms_per_position']:.4f} ms/position, "
          f"auto {inter['auto']['mean_ms_per_position']:.4f} ms/position ({inter['auto']['refreshes']} refreshes)",
          flush=True)
    del cache, op
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--plain-steps", type=int, default=400)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--cycles", type=int, default=40, help="extend-64 + step-1 cycles of the interleaved workload")
    ap.add_argument("--skip-operator", action="store_true")
    ap.add_argument("--skip-backbone", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import hyena_dna_b200 as H
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    ops = H.ops
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    Lmax, D, B = 1 << 20, 256, 1
    margin = max(args.windows * ops.WINDOW + ops.WINDOW_AFTER_STEPS + 8 + args.warmup, args.cycles * 65) + 64
    ts = (1 << 14, 1 << 17, Lmax - margin)
    ts_op = (1 << 14, 1 << 15, 1 << 16, 1 << 17, Lmax - margin)      # 2^15, 2^16: either side of WINDOW_MIN_T
    res = {"card": card(), "window": ops.WINDOW, "window_min_t": ops.WINDOW_MIN_T,
           "window_after_steps": ops.WINDOW_AFTER_STEPS, "windows": args.windows, "warmup": args.warmup}
    print("card:", res["card"])
    x = torch.randn(B, 1, D, device=dev, generator=gen)

    if not args.skip_operator:
        _operator(ops, args, res, ts_op, Lmax - margin, x, gen)

    if not args.skip_backbone:
        m = H.Backbone(D, args.layers, partial(H.HyenaOperator, l_max=Lmax, emb_dim=5),
                       mlp_cls=partial(H.Mlp, hidden_features=4 * D)).to(dev)
        cache = m.allocate_decode_cache(B, Lmax)
        for c in cache.layers:
            c.h.normal_(generator=gen)
            c.tail.normal_(generator=gen)
        with torch.no_grad():
            _model(ops, "backbone", m, cache, ts, x, args, res)
        res["backbone_layers"] = args.layers
        res["backbone_window_nbytes"] = cache.window_nbytes
    print("card:", res["card"])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
