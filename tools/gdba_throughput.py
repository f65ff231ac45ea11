#!/usr/bin/env python
"""GDBA throughput on the C4-shaped instance (generators.config_c4: 1M variables, d = 20, degree 6,
3M binary constraints with integer costs), f32 by default, increase modes T and E.

    python tools/gdba_throughput.py [--vars N] [--precision f32|f64] [--modes T,E] [--steps K] [--warmup W]
                                    [--repeats R]

For every increase mode, times fg_gdba_step (the two kernels of a round, no host work in between) with
CUDA events after `--warmup` rounds, `--repeats` times `--steps` rounds, and prints one JSON line: the
microseconds per round of every repeat and their median, the median variable-updates per second
(variables x rounds / s), the modifier storage (computed from the shapes), the card's name and its
power limit.  Exits non-zero without a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main(argv=None):
    ap = argparse.ArgumentParser(prog="gdba_throughput")
    ap.add_argument("--vars", type=int, default=1_000_000)
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--modes", default="T,E", help="comma-separated increase modes")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("gdba_throughput: no CUDA device (the GDBA engine runs on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200.engine import GdbaEngine
    from pydcop_b200.generators import config_c4
    from pydcop_b200.layout import layout_from_instance

    layout = layout_from_instance(config_c4(args.seed, n_vars=args.vars))
    out = {"workload": "gdba_c4", "n_vars": args.vars, "precision": args.precision, "steps": args.steps,
           "warmup": args.warmup, "launches_per_cycle": 2, "device": torch.cuda.get_device_name(),
           "power_limit_w": power_limit_w(), "modes": {}}
    for mode in args.modes.split(","):
        eng = GdbaEngine(layout, precision=args.precision, increase_mode=mode, seed=args.seed + 1).init()
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
        out["modes"][mode] = {"us_per_cycle": [round(x, 2) for x in us], "us_per_cycle_median": round(med, 2),
                              "var_updates_per_s": args.vars / (med * 1e-6), "modifier_bytes": eng.modifier_bytes}
        eng.close()
        del eng
        torch.cuda.empty_cache()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
