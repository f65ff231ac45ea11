#!/usr/bin/env python
"""What the device cost trace (engine start_trace, solve(trace=True)) and the best cycle kept with it
(start_trace(best=True), solve(best=True)) cost per cycle.

Three parts, each one JSON line with the card's name, power limit and SM clock:

1. `engines`: device time per cycle of the same engine stepped plain, with a trace attached, and with a trace that
   also keeps the best cycle, CUDA events around `--cycles` cycles after `--warmup`, the three arms alternating
   `--repeats` times (median and spread of each arm).  MaxSum on BASELINE.json's single-GPU configs (C2: 100k vars
   d=10 deg=4; C5: 50k arity-3 factors d=8) and DSA on C2 and C4's graph (1M vars d=20 deg=6) run on one GPU
   (`--cases` picks some of them).
2. `batch`: tools/batch_throughput.py's workload (`--problems` x random_factor_graph(100, 3, 150, 2), stop_cycle 100)
   through solve_batch plain, with trace=True and with trace=True and best=True, per batched family: wall time of each
   (median of `--repeats`, alternating), whether the results (assignment, status, cycle, cost, violation) are
   identical in all three, and the per-cycle device cost of one union engine in the three arms as in part 1.
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


def sm_clock_mhz():
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30)
        cur, top = (float(x) for x in r.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": cur, "sm_clock_max_mhz": top}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return {"sm_clock_mhz": None, "sm_clock_max_mhz": None}


def card():
    import torch
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(), **sm_clock_mhz()}


ARMS = ("plain", "traced", "best")   # no trace; a trace; a trace that also keeps the best cycle


def per_cycle_us(engine, cycles, warmup, arm, unary, seg=None):
    """Device microseconds per cycle of `cycles` engine.step(1) calls (the solve() loop steps in chunks; one call per
    cycle is the worst case for the host side and the same for every arm)."""
    import torch
    if arm != "plain":
        engine.start_trace(cycles + warmup, float("inf"), unary, seg, best=arm == "best")
    engine.step(warmup)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    engine.step(cycles)
    b.record()
    b.synchronize()
    if arm != "plain":
        assert len(engine.trace()["time"]) == cycles + warmup
        if arm == "best":
            assert (engine.best()["cycle"] >= 1).all()
        engine.stop_trace()
    return a.elapsed_time(b) * 1e3 / cycles


def engine_arms(make, unary, cycles, warmup, repeats, seg=None):
    """Alternating plain / traced / best runs of fresh engines from make(); median and range of each arm, in
    us/cycle."""
    arms = {arm: [] for arm in ARMS}
    for _ in range(repeats):
        for arm in ARMS:
            e = make()
            arms[arm].append(per_cycle_us(e, cycles, warmup, arm, unary, seg))
            e.close()
    out = {f"{k}_us_per_cycle": round(statistics.median(v), 2) for k, v in arms.items()}
    out.update({f"{k}_range_us": [round(min(v), 2), round(max(v), 2)] for k, v in arms.items()})
    out["overhead_us_per_cycle"] = round(out["traced_us_per_cycle"] - out["plain_us_per_cycle"], 2)
    out["overhead_pct"] = round(100 * out["overhead_us_per_cycle"] / out["plain_us_per_cycle"], 1)
    out["best_over_trace_us_per_cycle"] = round(out["best_us_per_cycle"] - out["traced_us_per_cycle"], 2)
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
    if args.cases:
        cases = [cases[int(i)] for i in args.cases.split(",")]
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
    from pydcop_b200.solve import _var_inputs, best_better, solve_batch
    dcops = problems(args.problems)
    families = args.families.split(",")
    keys = ("assignment", "status", "cycle", "cost", "violation")
    for kind in families:
        p = {"stop_cycle": 100}
        solve_batch(dcops[:20], kind, p, precision=args.precision, seed=1)     # warm-up, both arms
        solve_batch(dcops[:20], kind, p, precision=args.precision, seed=1, trace=True, best=True)
        times = {arm: [] for arm in ARMS}
        same = True
        for _ in range(args.repeats):
            for arm in ARMS:
                t = time.perf_counter()
                res = solve_batch(dcops, kind, p, precision=args.precision, seed=1, trace=arm != "plain",
                                  best=arm == "best")
                times[arm].append(time.perf_counter() - t)
                if arm == "plain":
                    want = [{k: r[k] for k in keys} for r in res]
                else:
                    same &= want == [{k: r[k] for k in keys} for r in res]
                    same &= all(len(r["trace"]["cycle"]) == len(res[0]["trace"]["cycle"]) > 0 for r in res)
                if arm == "best":
                    same &= all(r["best"] is not None and 1 <= r["best"]["cycle"] <= r["cycle"] for r in res)
                    # problems whose best cycle beats the last one, both as the trace recorded them (the result's
                    # own cost is summed in another order)
                    gains = sum(best_better(r["best"]["cost"], r["best"]["violation"], r["trace"]["cost"][-1],
                                            r["trace"]["violation"][-1], d.objective == "max")
                                for d, r in zip(dcops, res))
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
                              best_s=round(statistics.median(times["best"]), 4),
                              results_identical=bool(same), problems_best_before_last=int(gains),
                              union_engine=dev, **card())), flush=True)


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
    ap.add_argument("--cases", default="", help="engines part: comma-separated indices into its cases (default all)")
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
