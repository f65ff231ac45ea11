#!/usr/bin/env python
"""Many small problems: problems per second of sequential solve() calls against one solve_batch().

Workload: `--problems` (default 1000) random binary problems of pyDcop-benchmark size, each
`generators.random_factor_graph(100, 3, 150, 2, seed=i, noise=0)` (100 variables over 3 values, 150 binary constraints
with integer costs 0..9, no variable costs), `stop_cycle` 100, f32 by default.

    python tools/batch_throughput.py [--problems N] [--subset S] [--families maxsum,dsa,...] [--precision f32|f64]
                                     [--seeds R] [--sweep P [--repeats K]]

Per family, one JSON line: problems/s of sequential solve() calls, timed on the first `--subset` problems (default 50;
the subset size is in the line), problems/s of solve_batch() over all N problems, the speed-up, and whether the batch's
results on the subset equal the sequential ones (assignment, status and cycle exactly, cost and violation too: the
costs are integers).  Both are timed from the problems in memory to the result dicts, after one warm-up run of each
on the first problems.  The card's name and power limit are in every line.  Exits non-zero without a CUDA device:
there is no CPU path.

With `--seeds R` the workload is a seed sweep instead (pydcop batch's iterations): the first generated problem run R
times with seeds `--seed` + r, as R sequential solve() calls (timed on the first `--subset` seeds) against one
solve_batch() with one seed per run; the line reports runs/s of each and whether the subset's results are equal.

With `--sweep P` the workload is a parameter sweep (pydcop batch's parameter combinations): the N problems times P
parameter sets of the family (SWEEPS), run three ways: one solve_batch() with one parameter dict per problem, P
solve_batch() calls (one per set), and sequential solve() calls on the first `--subset` (problem, set) pairs.  The arms
run in turn, rotated over `--repeats` rounds; the line reports every arm's problems/s (the best round), the speed-up of
the one call over the P calls, and whether all three agree (the one call on every problem with the P calls, and on the
subset with solve()).
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gdba_throughput import power_limit_w  # noqa: E402

FAMILIES = ("maxsum", "dsa", "adsa", "mgm", "mgm2", "gdba", "mixeddsa")


def _spread(lo, hi, p):
    return [round(lo + (hi - lo) * k / max(p - 1, 1), 6) for k in range(p)]


# --sweep P: the parameter sets of each family, all inside one union
SWEEPS = {"dsa": lambda p: [{"probability": x} for x in _spread(0.1, 0.9, p)],
          "adsa": lambda p: [{"probability": x} for x in _spread(0.1, 0.9, p)],
          "mgm2": lambda p: [{"threshold": x} for x in _spread(0.1, 0.9, p)],
          "gdba": lambda p: [{"modifier": "AM"[k % 2], "violation": ("NZ", "NM", "MX")[k // 2 % 3]} for k in range(p)],
          "mixeddsa": lambda p: [{"proba_hard": x} for x in _spread(0.1, 0.9, p)],
          "maxsum": lambda p: [{"noise": x} for x in _spread(0.0, 0.05, p)]}


def problems(n, seed=0):
    from pydcop_b200 import ingest
    from pydcop_b200.generators import random_factor_graph
    return [ingest.from_arrays(random_factor_graph(100, 3, 150, 2, seed=seed + i, noise=0), name=f"p{i}") for i in range(n)]


def _same(r, s):
    return (r["assignment"] == s["assignment"] and (r["status"], r["cycle"], r["violation"], r["cost"])
            == (s["status"], s["cycle"], s["violation"], s["cost"]))


def main(argv=None):
    ap = argparse.ArgumentParser(prog="batch_throughput")
    ap.add_argument("--problems", type=int, default=1000)
    ap.add_argument("--subset", type=int, default=50)
    ap.add_argument("--families", default=",".join(FAMILIES))
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--stop-cycle", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0, help="the problems' generator seed and the runs' seed")
    ap.add_argument("--seeds", type=int, default=0, metavar="R",
                    help="seed sweep: one problem solved with R seeds (--seed + r) instead of --problems problems")
    ap.add_argument("--sweep", type=int, default=0, metavar="P",
                    help="parameter sweep: every problem with P parameter sets, one call against P calls")
    ap.add_argument("--repeats", type=int, default=2, help="--sweep: rounds of the three arms")
    args = ap.parse_args(argv)
    families = args.families.split(",")
    for f in families:
        if f not in FAMILIES:
            ap.error(f"unknown family {f!r}: expected some of {','.join(FAMILIES)}")
    if args.seeds > 0:
        return sweep(args, families)
    if args.sweep > 0:
        bad = [f for f in families if f not in SWEEPS]
        if bad:
            ap.error(f"--sweep: no parameter sweep for {','.join(bad)}")
        return param_sweep(args, families)
    subset = min(args.subset, args.problems)
    dcops = problems(args.problems, args.seed)

    import torch
    if not torch.cuda.is_available():
        print("batch_throughput: no CUDA device (the engines run on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.solve import solve, solve_batch

    card, watts = torch.cuda.get_device_name(), power_limit_w()
    for kind in families:
        p = {"stop_cycle": args.stop_cycle}
        run = lambda d: solve(d, kind, p, precision=args.precision, seed=args.seed)  # noqa: E731
        run(dcops[0])                                   # warm-up: module loads, allocator
        solve_batch(dcops[:4], kind, p, precision=args.precision, seed=args.seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seq = [run(d) for d in dcops[:subset]]
        t_seq = time.perf_counter() - t0
        t0 = time.perf_counter()
        res = solve_batch(dcops, kind, p, precision=args.precision, seed=args.seed)
        t_batch = time.perf_counter() - t0
        print(json.dumps({"workload": "random_factor_graph(100, 3, 150, 2, noise=0)", "family": kind,
                          "precision": args.precision, "stop_cycle": args.stop_cycle, "problems": args.problems,
                          "sequential_subset": subset, "sequential_problems_per_s": subset / t_seq,
                          "batch_problems_per_s": args.problems / t_batch,
                          "speedup": (args.problems / t_batch) / (subset / t_seq),
                          "batch_ingest_s": res[0]["ingest_time"], "batch_s": t_batch,
                          "equal_on_subset": all(_same(r, s) for r, s in zip(res[:subset], seq)),
                          "device": card, "power_limit_w": watts}), flush=True)
    return 0


def sweep(args, families):
    """The --seeds leg: problem 0 run with seeds --seed + r, r < R, sequentially (first --subset seeds) and batched."""
    subset = min(args.subset, args.seeds)
    d = problems(1, args.seed)[0]
    seeds = [args.seed + r for r in range(args.seeds)]

    import torch
    if not torch.cuda.is_available():
        print("batch_throughput: no CUDA device (the engines run on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.solve import solve, solve_batch

    card, watts = torch.cuda.get_device_name(), power_limit_w()
    for kind in families:
        p = {"stop_cycle": args.stop_cycle}
        run = lambda s: solve(d, kind, p, precision=args.precision, seed=s)  # noqa: E731
        run(seeds[0])                                   # warm-up: module loads, allocator
        solve_batch([d] * 2, kind, p, precision=args.precision, seed=[seeds[0], seeds[0] + 1])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seq = [run(s) for s in seeds[:subset]]
        t_seq = time.perf_counter() - t0
        t0 = time.perf_counter()
        res = solve_batch([d] * args.seeds, kind, p, precision=args.precision, seed=seeds)
        t_batch = time.perf_counter() - t0
        print(json.dumps({"workload": "random_factor_graph(100, 3, 150, 2, noise=0) x seeds", "family": kind,
                          "precision": args.precision, "stop_cycle": args.stop_cycle, "seeds": args.seeds,
                          "sequential_subset": subset, "sequential_runs_per_s": subset / t_seq,
                          "batch_runs_per_s": args.seeds / t_batch,
                          "speedup": (args.seeds / t_batch) / (subset / t_seq),
                          "batch_ingest_s": res[0]["ingest_time"], "batch_s": t_batch,
                          "equal_on_subset": all(_same(r, s) for r, s in zip(res[:subset], seq)),
                          "distinct_assignments": len({tuple(sorted(r["assignment"].items())) for r in res}),
                          "device": card, "power_limit_w": watts}), flush=True)
    return 0


def param_sweep(args, families):
    """The --sweep leg: N problems x P parameter sets, as one call, P calls and sequential solve() on a subset."""
    dcops = problems(args.problems, args.seed)
    import torch
    if not torch.cuda.is_available():
        print("batch_throughput: no CUDA device (the engines run on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.solve import solve, solve_batch

    card, watts = torch.cuda.get_device_name(), power_limit_w()
    n, P = len(dcops), args.sweep
    subset = min(args.subset, n * P)
    for kind in families:
        sets = [dict(s, stop_cycle=args.stop_cycle) for s in SWEEPS[kind](P)]
        probs = [d for d in dcops for _ in sets]           # problem-major, then set
        params = [s for _ in dcops for s in sets]
        kw = dict(precision=args.precision, seed=args.seed)
        solve(dcops[0], kind, sets[0], **kw)               # warm-up: module loads, allocator
        solve_batch(probs[:2 * P], kind, params[:2 * P], **kw)
        best = {"one": float("inf"), "per_set": float("inf"), "sequential": float("inf")}
        out = {}

        def one():
            out["one"] = solve_batch(probs, kind, params, **kw)

        def per_set():
            res = [None] * len(probs)
            for j, s in enumerate(sets):
                for i, r in enumerate(solve_batch(dcops, kind, s, **kw)):
                    res[i * P + j] = r
            out["per_set"] = res

        def sequential():
            out["sequential"] = [solve(d, kind, s, **kw) for d, s in zip(probs[:subset], params[:subset])]

        arms = [("one", one), ("per_set", per_set), ("sequential", sequential)]
        for k in range(max(1, args.repeats)):
            for name, fn in arms[k % 3:] + arms[:k % 3]:   # rotated, so no arm always runs first
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                best[name] = min(best[name], time.perf_counter() - t0)
        equal = (all(_same(r, s) for r, s in zip(out["one"], out["per_set"]))
                 and all(_same(r, s) for r, s in zip(out["one"][:subset], out["sequential"])))
        print(json.dumps({"workload": "random_factor_graph(100, 3, 150, 2, noise=0) x parameter sets", "family": kind,
                          "precision": args.precision, "stop_cycle": args.stop_cycle, "problems": n, "sets": P,
                          "sweep": [{k: v for k, v in s.items() if k != "stop_cycle"} for s in sets],
                          "one_call_problems_per_s": n * P / best["one"],
                          "per_set_calls_problems_per_s": n * P / best["per_set"],
                          "sequential_subset": subset, "sequential_problems_per_s": subset / best["sequential"],
                          "speedup_one_vs_per_set": best["per_set"] / best["one"],
                          "one_call_ingest_s": out["one"][0]["ingest_time"], "repeats": args.repeats,
                          "all_equal": equal, "device": card, "power_limit_w": watts}), flush=True)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
