#!/usr/bin/env python
"""Many small problems: problems per second of sequential solve() calls against one solve_batch().

Workload: `--problems` (default 1000) random binary problems of pyDcop-benchmark size, each
`generators.random_factor_graph(100, 3, 150, 2, seed=i, noise=0)` (100 variables over 3 values, 150 binary constraints
with integer costs 0..9, no variable costs), `stop_cycle` 100, f32 by default.

    python tools/batch_throughput.py [--problems N] [--subset S] [--families maxsum,dsa,...] [--precision f32|f64]
                                     [--seeds R]

Per family, one JSON line: problems/s of sequential solve() calls, timed on the first `--subset` problems (default 50;
the subset size is in the line), problems/s of solve_batch() over all N problems, the speed-up, and whether the batch's
results on the subset equal the sequential ones (assignment, status and cycle exactly, cost and violation too: the
costs are integers).  Both are timed from the problems in memory to the result dicts, after one warm-up run of each
on the first problems.  The card's name and power limit are in every line.  Exits non-zero without a CUDA device:
there is no CPU path.

With `--seeds R` the workload is a seed sweep instead (pydcop batch's iterations): the first generated problem run R
times with seeds `--seed` + r, as R sequential solve() calls (timed on the first `--subset` seeds) against one
solve_batch() with one seed per run; the line reports runs/s of each and whether the subset's results are equal.
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
    args = ap.parse_args(argv)
    families = args.families.split(",")
    for f in families:
        if f not in FAMILIES:
            ap.error(f"unknown family {f!r}: expected some of {','.join(FAMILIES)}")
    if args.seeds > 0:
        return sweep(args, families)
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


if __name__ == "__main__":
    raise SystemExit(main())
