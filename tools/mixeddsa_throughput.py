#!/usr/bin/env python
"""MixedDSA throughput on a hard-colouring-plus-soft-cost instance: `--vars` variables over 4 colours, 2.25 x vars
binary constraints (mean degree 4.5), half of them hard `!=` (+inf on equal colours, integer costs 0..3 elsewhere),
the others soft integer tables, and dyadic variable costs; f32 by default.

    python tools/mixeddsa_throughput.py [--vars N] [--precision f32|f64] [--steps K] [--warmup W] [--repeats R]

Times fg_mixeddsa_step (one kernel per round) with CUDA events after `--warmup` rounds, `--repeats` times `--steps`
rounds, and prints one JSON line: the microseconds per round of every repeat and their median, the median rounds per
second, the card's name and its power limit.  Exits non-zero without a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from gdba_throughput import power_limit_w  # noqa: E402


def instance(n, seed, dom=4, degree=4.5):
    import numpy as np
    from pydcop_b200.layout import default_var_csr
    rng = np.random.default_rng(seed)
    m = int(n * degree / 2)
    a = rng.integers(0, n, m)
    b = (a + rng.integers(1, n, m)) % n            # distinct endpoints
    t = rng.integers(0, 4, (m, dom, dom)).astype(np.float64)
    hard = rng.random(m) < 0.5
    for x in range(dom):
        t[hard, x, x] = np.inf
    inst = dict(dom_size=np.full(n, dom, dtype=np.int32), factor_ptr=np.arange(0, 2 * m + 1, 2, dtype=np.int64),
                edge_var=np.stack([a, b], 1).reshape(-1).astype(np.int32), tables=t.reshape(-1),
                unary=np.floor(rng.uniform(0, 8, n * dom)) / 8.0)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    return inst


def main(argv=None):
    ap = argparse.ArgumentParser(prog="mixeddsa_throughput")
    ap.add_argument("--vars", type=int, default=1_000_000)
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("mixeddsa_throughput: no CUDA device (the MixedDSA engine runs on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.engine import MixedDsaEngine
    from pydcop_b200.layout import layout_from_instance

    layout = layout_from_instance(instance(args.vars, args.seed))
    eng = MixedDsaEngine(layout, precision=args.precision, seed=args.seed + 1).init()
    eng.step(args.warmup)
    torch.cuda.synchronize()
    us = []
    for _ in range(args.repeats):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        eng.step(args.steps)
        t1.record()
        t1.synchronize()
        us.append(t0.elapsed_time(t1) * 1e3 / args.steps)
    med = sorted(us)[len(us) // 2]
    cost, violations = eng.solution_cost()
    print(json.dumps({"workload": "mixeddsa_hard_colouring", "n_vars": args.vars, "n_factors": layout.n_factors,
                      "precision": args.precision, "steps": args.steps, "warmup": args.warmup,
                      "launches_per_cycle": 1, "device": torch.cuda.get_device_name(),
                      "power_limit_w": power_limit_w(), "us_per_cycle": [round(x, 2) for x in us],
                      "us_per_cycle_median": round(med, 2), "rounds_per_s": 1e6 / med,
                      "violations_after": violations, "soft_cost_after": cost}))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
