#!/usr/bin/env python
"""DPOP device throughput on two workloads (pydcop_b200.generators.bounded_separator_instance):
    deep  ~10^6 variables, d = 10, small separators: the light-path (one warp per segment) kernel
    wide  300 variables, separators of 6 at d = 10: joined tables of 10^7 entries on the grid-wide kernel
For each: the tree actually built (max separator, height, rounds, launches, big nodes, arena bytes), the
host tree build, the device time of the UTIL and VALUE phases (CUDA events around the whole run and around
the VALUE launches alone, best of --repeat runs), joined-entry candidates per second, the bytes the UTIL
phase reads and writes (computed from the shapes) against the H100 SXM's 3.35 TB/s, and the end-to-end
solve() time on the same instance.  Prints the card name and power limit read in the same run.

    python tools/dpop_throughput.py [--precision f32|f64] [--repeat 5] [--deep-vars 1000000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def shape_counts(t, eng):
    """Joined-entry candidates (UTIL entries x own domain) and UTIL-phase bytes: every term read once per
    candidate, every UTIL entry written once."""
    d = eng.layout.canon_dom_size.astype(np.int64)
    elem = np.dtype(eng.np_dtype).itemsize
    tp = eng.dev["term_ptr"].cpu().numpy()
    n_terms = np.diff(tp)
    util = np.array(t.util_size, dtype=np.float64)
    cand = float((util * d).sum())
    read = float((util * d * (1 + n_terms)).sum()) * elem
    write = float(util.sum()) * elem
    return cand, read, write


def run(name, inst, precision, repeat):
    import torch
    from pydcop_b200 import pseudotree as pt, solve as S
    from pydcop_b200.engine import DpopEngine
    from pydcop_b200.layout import build_layout
    t0 = time.perf_counter()
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    t_tree = time.perf_counter() - t0
    L = build_layout(**inst)
    t1 = time.perf_counter()
    eng = DpopEngine(L, t, precision=precision)
    t_engine = time.perf_counter() - t1
    s = eng.sched
    lib, h, st = eng.lib, eng._h, eng._stream()
    full, val = [], []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    lib.fg_dpop_run(h, st)                         # warm-up
    torch.cuda.synchronize()
    for _ in range(repeat):
        ev[0].record()
        eng._check(lib.fg_dpop_run(h, st), "fg_dpop_run")
        ev[1].record()
        torch.cuda.synchronize()
        full.append(ev[0].elapsed_time(ev[1]) * 1e-3)
    # the VALUE phase alone: an engine whose UTIL launch list is empty reads the arena the runs above left
    d = eng._desc
    saved = d.n_util_launches
    d.n_util_launches = 0
    import ctypes as C
    hv = C.c_void_p()
    eng._check(lib.fg_dpop_create(C.byref(d), C.byref(hv)), "fg_dpop_create")
    d.n_util_launches = saved
    lib.fg_dpop_run(hv, st)
    torch.cuda.synchronize()
    for _ in range(repeat):
        ev[0].record()
        lib.fg_dpop_run(hv, st)
        ev[1].record()
        torch.cuda.synchronize()
        val.append(ev[0].elapsed_time(ev[1]) * 1e-3)
    lib.fg_dpop_destroy(hv)
    t_full, t_val = min(full), min(val)
    t_util = t_full - t_val
    cand, rd, wr = shape_counts(t, eng)
    max_sep = max((len(x) for x in t.sep), default=0)
    del eng
    torch.cuda.empty_cache()
    t2 = time.perf_counter()
    res = S.solve(dict(inst), "dpop", precision=precision)
    t_solve = time.perf_counter() - t2
    return dict(workload=name, n_vars=t.n_vars, max_separator=max_sep, tree_height=t.height, rounds=s.rounds,
                launches=s.n_launches, big_nodes=len(s.big_nodes), arena_bytes=int(sum(t.util_size)) * (8 if precision == "f64" else 4),
                host_tree_build_s=round(t_tree, 3), engine_setup_s=round(t_engine, 3),
                util_ms=round(t_util * 1e3, 3), value_ms=round(t_val * 1e3, 3),
                joined_candidates_per_s=cand / t_util if t_util > 0 else None,
                util_bytes_read=rd, util_bytes_written=wr,
                util_hbm_fraction=(rd + wr) / t_util / HBM_BYTES_PER_S if t_util > 0 else None,
                solve_s=round(t_solve, 3), solve_status=res["status"], solve_cost=res["cost"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f64", choices=["f32", "f64"])
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--deep-vars", type=int, default=1_000_000)
    a = ap.parse_args()
    from pydcop_b200.generators import bounded_separator_instance
    print(json.dumps({"card": card(), "precision": a.precision}))
    work = {"deep": lambda: bounded_separator_instance(a.deep_vars, 10, back=2, span=3, p_back=0.3, seed=1),
            "wide": lambda: bounded_separator_instance(300, 10, back=5, span=1, seed=2)}
    for name, make in work.items():
        print(json.dumps(run(name, make(), a.precision, a.repeat)), flush=True)


if __name__ == "__main__":
    main()
