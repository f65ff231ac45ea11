#!/usr/bin/env python
"""What the device cost trace (engine start_trace, solve(trace=True)) costs per cycle.

Three parts, each one JSON line with the card's name and power limit:

1. `engines`: device time per cycle of the same engine stepped with and without a trace attached, CUDA events around
   `--cycles` cycles after `--warmup`, the two arms alternating `--repeats` times (median and spread of each arm).
   MaxSum on BASELINE.json's single-GPU configs (C2: 100k vars d=10 deg=4; C5: 50k arity-3 factors d=8) and DSA on C2
   and C4's graph (1M vars d=20 deg=6) run on one GPU.
2. `batch`: tools/batch_throughput.py's workload (`--problems` x random_factor_graph(100, 3, 150, 2), stop_cycle 100)
   through solve_batch with and without trace=True, per batched family: wall time of each (median of `--repeats`,
   alternating), whether the results (assignment, status, cycle, cost, violation) are identical, and the per-cycle
   device cost of one union engine with and without a trace as in part 1.
3. `metrics_every_1`: wall time of the CLI's host-side metrics at every cycle (solve(chunk=1, on_cycle=...) with the
   numpy solution_cost, what `--run_metrics --metrics_every 1` does) against solve(trace=True), on C2 with MaxSum.

    python tools/trace_overhead.py [--parts engines,batch,metrics_every_1] [--cycles N] [--repeats R]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gdba_throughput import power_limit_w  # noqa: E402


def card():
    import torch
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}


def per_cycle_us(engine, cycles, warmup, traced, unary, seg=None):
    """Device microseconds per cycle of `cycles` engine.step(1) calls (the solve() loop steps in chunks; one call per
    cycle is the worst case for the host side and the same for both arms)."""
    import torch
    if traced:
        engine.start_trace(cycles + warmup, float("inf"), unary, seg)
    engine.step(warmup)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    engine.step(cycles)
    b.record()
    b.synchronize()
    if traced:
        assert len(engine.trace()["time"]) == cycles + warmup
        engine.stop_trace()
    return a.elapsed_time(b) * 1e3 / cycles


def engine_arms(make, unary, cycles, warmup, repeats, seg=None):
    """Alternating plain / traced runs of fresh engines from make(); median and range of each arm, in us/cycle."""
    arms = {"plain": [], "traced": []}
    for _ in range(repeats):
        for arm in ("plain", "traced"):
            e = make()
            arms[arm].append(per_cycle_us(e, cycles, warmup, arm == "traced", unary, seg))
            e.close()
    out = {f"{k}_us_per_cycle": round(statistics.median(v), 2) for k, v in arms.items()}
    out.update({f"{k}_range_us": [round(min(v), 2), round(max(v), 2)] for k, v in arms.items()})
    out["overhead_us_per_cycle"] = round(out["traced_us_per_cycle"] - out["plain_us_per_cycle"], 2)
    out["overhead_pct"] = round(100 * out["overhead_us_per_cycle"] / out["plain_us_per_cycle"], 1)
    return out


def part_engines(args):
    import numpy as np
    from pydcop_b200 import generators as G
    from pydcop_b200.engine import make_engine
    from pydcop_b200.layout import build_layout
    cases = [("maxsum", "C2 100k vars d=10 deg=4", lambda: G.config_c2(0)),
             ("maxsum", "C5 50k arity-3 factors d=8", lambda: G.config_c5(0)),
             ("dsa", "C2 100k vars d=10 deg=4", lambda: G.config_c2(0)),
             ("dsa", "C4 1M vars d=20 deg=6 on one GPU", lambda: G.config_c4(0))]
    for kind, name, gen in cases:
        inst = gen()
        L = build_layout(**inst)
        unary = np.asarray(inst["unary"], dtype=np.float64)
        res = engine_arms(lambda: make_engine(kind, L, {}, precision=args.precision, seed=1).init(), unary,
                          args.cycles, args.warmup, args.repeats)
        print(json.dumps(dict(part="engines", algo=kind, workload=name, precision=args.precision, **res, **card())),
              flush=True)


def part_batch(args):
    from batch_throughput import problems
    from pydcop_b200 import batch
    from pydcop_b200.engine import make_engine
    from pydcop_b200.solve import _var_inputs, solve_batch
    dcops = problems(args.problems)
    families = args.families.split(",")
    keys = ("assignment", "status", "cycle", "cost", "violation")
    for kind in families:
        p = {"stop_cycle": 100}
        solve_batch(dcops[:20], kind, p, precision=args.precision, seed=1)     # warm-up, both arms
        solve_batch(dcops[:20], kind, p, precision=args.precision, seed=1, trace=True)
        times = {"plain": [], "traced": []}
        same = True
        for _ in range(args.repeats):
            for arm in ("plain", "traced"):
                t = time.perf_counter()
                res = solve_batch(dcops, kind, p, precision=args.precision, seed=1, trace=arm == "traced")
                times[arm].append(time.perf_counter() - t)
                if arm == "plain":
                    want = [{k: r[k] for k in keys} for r in res]
                else:
                    same &= want == [{k: r[k] for k in keys} for r in res]
                    same &= all(len(r["trace"]["cycle"]) == len(res[0]["trace"]["cycle"]) > 0 for r in res)
        members = list(range(len(dcops)))
        u = batch.build_union(dcops, members, lambda d: _var_inputs(kind, d, "min"), 0.0, 1)
        L = batch.union_layout(u, dcops)
        seg = (u.seg_factor, u.seg_var, len(members))
        dev = engine_arms(lambda: make_engine(kind, L, {}, precision=args.precision, seed=1, var_rank=u.var_rank,
                                              isolated_value=u.isolated_value, var_global_id=u.var_global_id).init(),
                          u.unary, args.cycles, args.warmup, args.repeats, seg)
        print(json.dumps(dict(part="batch", algo=kind, problems=len(dcops), precision=args.precision,
                              plain_s=round(statistics.median(times["plain"]), 4),
                              traced_s=round(statistics.median(times["traced"]), 4),
                              results_identical=bool(same), union_engine=dev, **card())), flush=True)


def part_metrics_every_1(args):
    from pydcop_b200 import generators as G
    from pydcop_b200 import ingest
    from pydcop_b200.solve import solution_cost, solve
    d = ingest.from_arrays(G.config_c2(0))
    n = args.metric_cycles
    p = {"stop_cycle": n}
    solve(d, "maxsum", {"stop_cycle": 5}, precision=args.precision, seed=1, trace=True)   # warm-up
    rows = []

    def collect(cycle, idx):
        rows.append(solution_cost(d, idx))
    t = time.perf_counter()
    solve(d, "maxsum", p, precision=args.precision, seed=1, chunk=1, on_cycle=collect)
    host = time.perf_counter() - t
    t = time.perf_counter()
    res = solve(d, "maxsum", p, precision=args.precision, seed=1, trace=True)
    dev = time.perf_counter() - t
    t = time.perf_counter()
    solve(d, "maxsum", p, precision=args.precision, seed=1)
    plain = time.perf_counter() - t
    import numpy as np
    host_cost = np.array([c for _, c in rows])
    same_viol = [v for v, _ in rows] == res["trace"]["violation"]
    rel = float(np.max(np.abs(host_cost - res["trace"]["cost"]) / np.maximum(np.abs(host_cost), 1e-300)))
    print(json.dumps(dict(part="metrics_every_1", algo="maxsum", workload="C2 100k vars d=10 deg=4", cycles=n,
                          precision=args.precision, host_metrics_every_1_s=round(host, 3),
                          device_trace_s=round(dev, 3), no_metrics_s=round(plain, 3),
                          violations_equal=same_viol, max_rel_cost_diff=rel, **card())), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="trace_overhead")
    ap.add_argument("--parts", default="engines,batch,metrics_every_1")
    ap.add_argument("--cycles", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--problems", type=int, default=1000)
    ap.add_argument("--families", default="maxsum,dsa,adsa,mgm,mgm2,gdba,mixeddsa")
    ap.add_argument("--metric-cycles", type=int, default=100)
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        print("trace_overhead: no CUDA device (there is no CPU path)", file=sys.stderr)
        return 1
    for part in args.parts.split(","):
        {"engines": part_engines, "batch": part_batch, "metrics_every_1": part_metrics_every_1}[part](args)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
