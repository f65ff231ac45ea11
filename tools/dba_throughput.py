#!/usr/bin/env python
"""DBA throughput on a random graph-colouring CSP: 1M variables, 4 colours, mean degree 4.5 (2.25M binary
constraints, `inf` where the two colours are equal, 0 elsewhere), generated from --seed; f32 by default.

    python tools/dba_throughput.py [--vars N] [--precision f32|f64] [--max-distance M] [--steps K] [--warmup W]
                                   [--repeats R]

Times fg_dba_step (the two kernels of a round, no host work in between) with CUDA events after `--warmup` rounds,
`--repeats` times `--steps` rounds, and prints one JSON line: the microseconds per round of every repeat and their
median, rounds per second, the bit-row bytes, the bytes a round reads and writes (computed from the shapes, see
`bytes_per_round`), the card's name and its power limit.  max_distance defaults to 0 so that no variable stops and
every measured round does the full work; the JSON says whether the engine finished.  Exits non-zero without a CUDA
device: there is no CPU path.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from gdba_throughput import power_limit_w  # noqa: E402


def colouring_csp(n_vars, d=4, degree=4.5, seed=0):
    """Random graph colouring: n_vars * degree / 2 constraints between two distinct random variables."""
    rng = np.random.default_rng(seed)
    m = int(round(n_vars * degree / 2))
    a = rng.integers(0, n_vars, m)
    b = (a + rng.integers(1, n_vars, m)) % n_vars
    t = np.where(np.eye(d, dtype=bool), np.inf, 0.0).reshape(-1)
    return dict(dom_size=np.full(n_vars, d, np.int32), factor_ptr=np.arange(0, 2 * m + 1, 2, dtype=np.int64),
                edge_var=np.stack([a, b], 1).reshape(-1).astype(np.int32), tables=np.tile(t, m))


def bytes_per_round(layout, nbr_entries):
    """Bytes the ok and improve kernels read and write in one round with every variable live, each element counted
    once, every move and weight raise counted: per variable 76 (ok) + 66 (improve, with the move); per neighbour
    entry 8 (ok: index, finish phase) + 32 (improve: index, finish phase, counter, improve, eval, rank); per slot
    29 + 4 per word of the one row it reads (ok: edge, class, other variable and its value, offset, row, weight,
    violated) + 9 (improve: weight read and write, violated)."""
    V, S = layout.n_vars, layout.n_edges
    row_words = (layout.dom_size[layout.slot_var].astype(np.int64) + 31) // 32
    return V * (76 + 66) + nbr_entries * (8 + 32) + S * (29 + 9) + 4 * int(row_words.sum())


def main(argv=None):
    ap = argparse.ArgumentParser(prog="dba_throughput")
    ap.add_argument("--vars", type=int, default=1_000_000)
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--max-distance", type=int, default=0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("dba_throughput: no CUDA device (the DBA engine runs on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.engine import DbaEngine
    from pydcop_b200.layout import layout_from_instance

    layout = layout_from_instance(colouring_csp(args.vars, seed=args.seed))
    eng = DbaEngine(layout, precision=args.precision, max_distance=args.max_distance, seed=args.seed + 1).init()
    nbr = int(eng.nbr_ptr[-1].item())
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
    bpr = bytes_per_round(layout, nbr)
    table_bytes = int(layout.tables.size) * np.dtype(eng.np_dtype).itemsize
    print(json.dumps({
        "workload": "dba_colouring_csp", "n_vars": args.vars, "n_constraints": layout.n_factors, "colours": 4,
        "precision": args.precision, "max_distance": args.max_distance, "steps": args.steps, "warmup": args.warmup,
        "launches_per_round": 2, "device": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(),
        "us_per_round": [round(x, 2) for x in us], "us_per_round_median": round(med, 2),
        "rounds_per_s": round(1e6 / med, 1), "var_updates_per_s": args.vars / (med * 1e-6),
        "bit_row_bytes": eng.bit_row_bytes, "table_bytes": table_bytes, "bytes_per_round": bpr,
        "gb_per_s_at_bytes_per_round": round(bpr / (med * 1e-6) / 1e9, 1),
        "finished": eng.finished, "cycle": eng.cycle, "unresolved": eng.unresolved}))
    eng.close()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
