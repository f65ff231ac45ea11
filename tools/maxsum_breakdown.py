#!/usr/bin/env python
"""Where a MaxSum cycle's time goes on the bench workload (C2: generators.config_c2, seed 0), and what the 8-bit
table copy of the factor side (DESIGN.md §3) changes.

    python tools/maxsum_breakdown.py [--workload c2|target] [--precision f32|f64] [--steps K] [--warmup W]
                                     [--repeats R] [--variants int8,full] [--no-profile] [--out FILE]

Two instances of identical shape and access pattern:
  int8  the instance as generated: integer tables in [0, 9], read by the factor kernel as 8-bit codes;
  full  the same instance with every table entry + 128: still integers, but out of int8 range, so the factor
        kernel reads them at full width.
For each, alternating, `--repeats` times: `--steps` cycles, CUDA events around every cycle on the launching
stream with a 256 MiB L2 flush outside the event pairs, after `--warmup` cycles (the rules of bench.py).
Then, in a run of its own, torch.profiler with CUDA activities gives the device time per launch of k_f2v_warp
and k_v2f_warp, once with the two sides on two streams and once serialised (PYDCOP_B200_SERIAL=1).  Prints one
JSON line: the per-repeat times, their spread, the kernel times, the algorithmic bytes per cycle (tables at the
value width, generators.algorithmic_bytes_per_cycle) beside the bytes actually stored and read (tables at the
width table_widths() reports), and the card's name and power limit.  Exits non-zero without a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    """Card name and power limit (query only)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                            os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30)
        name, pl = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def stored_bytes(L, eng, w):
    """Algorithmic bytes per cycle with every class's tables counted at the width the factor kernel reads."""
    from pydcop_b200.generators import algorithmic_bytes_per_cycle
    b = algorithmic_bytes_per_cycle(L, w)
    for c, tw in zip(L.classes, eng.table_widths()):
        b -= c.n_factors * c.table_size * (w - tw)
    return b


def time_steps(eng, flush, steps):
    import torch
    evs = []
    for _ in range(steps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.step(1)
        b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    return 1e3 * sum(a.elapsed_time(b) for a, b in evs) / steps   # us per cycle


def kernel_times(L, precision, steps, serial):
    """Device time per launch (us) of the two warp kernels, from torch.profiler, in a run of their own."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from pydcop_b200.engine import MaxSumEngine
    old = os.environ.get("PYDCOP_B200_SERIAL")
    if serial:
        os.environ["PYDCOP_B200_SERIAL"] = "1"
    try:
        eng = MaxSumEngine(L, precision=precision).init()
    finally:
        if old is None:
            os.environ.pop("PYDCOP_B200_SERIAL", None)
        else:
            os.environ["PYDCOP_B200_SERIAL"] = old
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    eng.step(5)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            flush.zero_()
            eng.step(1)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in ("k_f2v_warp", "k_v2f_warp"):
            if k in ev.key and ev.count:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[k] = round(t / ev.count, 2)
    eng.close()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="maxsum_breakdown")
    ap.add_argument("--workload", default="c2", choices=["c2", "target"])
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--variants", default="int8,full")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        print("maxsum_breakdown: no CUDA device (the engine runs on the GPU only)", file=sys.stderr)
        return 2
    from pydcop_b200 import build_layout
    from pydcop_b200.engine import MaxSumEngine
    from pydcop_b200 import generators as G

    inst = G.config_c2(seed=0) if args.workload == "c2" else G.config_target()
    variants = [v for v in args.variants.split(",") if v]
    w = 4 if args.precision == "f32" else 8
    res = {"workload": args.workload, "precision": args.precision, "steps": args.steps, "warmup": args.warmup,
           "repeats": args.repeats, "env": {k: v for k, v in os.environ.items() if k.startswith("PYDCOP_B200_")}}
    layouts, engines = {}, {}
    for v in variants:
        iv = dict(inst)
        if v == "full":
            iv["tables"] = np.asarray(inst["tables"]) + np.float32(128)
        L = build_layout(**iv)
        eng = MaxSumEngine(L, precision=args.precision, record_sent=True).init()
        layouts[v], engines[v] = L, eng
        res[v] = {"table_widths": sorted(set(eng.table_widths())),
                  "algorithmic_bytes_per_cycle": G.algorithmic_bytes_per_cycle(L, w),
                  "stored_bytes_per_cycle": stored_bytes(L, eng, w), "us_per_cycle": []}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for v in variants:
        engines[v].step(max(3, args.warmup))
    torch.cuda.synchronize()
    for _ in range(args.repeats):
        for v in variants:   # alternating: drifts of the shared machine hit both alike
            res[v]["us_per_cycle"].append(round(time_steps(engines[v], flush, args.steps), 2))
    for v in variants:
        us = res[v]["us_per_cycle"]
        res[v]["us_min_max"] = [min(us), max(us)]
        res[v]["us_median"] = sorted(us)[len(us) // 2]
        engines[v].close()
    if "int8" in res and "full" in res:
        res["int8_over_full"] = round(res["int8"]["us_median"] / res["full"]["us_median"], 4)
    if not args.no_profile:
        for v in variants:
            res[v]["kernel_us_concurrent"] = kernel_times(layouts[v], args.precision, 50, serial=False)
            res[v]["kernel_us_serial"] = kernel_times(layouts[v], args.precision, 50, serial=True)
    res["device"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
