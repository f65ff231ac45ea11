#!/usr/bin/env python
"""SyncBB messages per second on the device, against the Python oracle on the host.

    python tools/syncbb_throughput.py [--precision f64] [--vars 29] [--constraints 44] [--seed 6]

The default instance (29 variables, 3 values, 44 random binary constraints with uniform costs in [0, 10) and 2 % inf
entries, names shuffled) needs 7.57 * 10^6 messages.  The whole search runs in launches of --chunk messages timed
with CUDA events; the card's name and power limit are read in the same run.  The host rate is the oracle
(tests/_syncbb_oracle.py) on the first --host-steps messages of the same search, and the same step functions the
kernel runs (csrc/syncbb_kernels.cuh through tests/hostshim/syncbb_host.cpp, built with `g++ -O2` in a temporary
directory) over the whole search on one CPU core.  SyncBB is a token walk: one CTA delivers one message at a time, so
the device rate is bound by the latency of one step, not by bandwidth.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def instance(n, n_cons, seed, p_inf=0.02, d=3):
    """Random binary constraints over shuffled names (var_rank a permutation), domains 1..d."""
    rng = np.random.default_rng(seed)
    pairs = [tuple(int(x) for x in rng.choice(n, 2, replace=False)) for _ in range(n_cons)]
    dom = rng.integers(1, d + 1, size=n).astype(np.int32)
    tabs = []
    for a, b in pairs:
        t = rng.random(dom[a] * dom[b]) * 10
        tabs.append(np.where(rng.random(t.size) < p_inf, np.inf, t))
    return dict(dom_size=dom, factor_ptr=np.arange(0, 2 * len(pairs) + 1, 2, dtype=np.int64),
                edge_var=np.array(pairs, dtype=np.int32).reshape(-1), tables=np.concatenate(tabs),
                var_rank=rng.permutation(n).astype(np.int32))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        return float(out[0]) if out else None
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def one_core_rate(inst, precision):
    """Messages/s of the kernel's step functions compiled for the host, whole search, one thread; None without g++."""
    from pydcop_b200 import _cabi
    from pydcop_b200.engine import fill_desc, host_state, syncbb_plan
    from pydcop_b200.layout import layout_from_instance
    src = os.path.join(ROOT, "tests", "hostshim", "syncbb_host.cpp")
    with tempfile.TemporaryDirectory() as td:
        so = os.path.join(td, "syncbb_host.so")
        try:
            subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src],
                           check=True, capture_output=True)
        except (OSError, subprocess.CalledProcessError):
            return None
        lib = C.CDLL(so)
        lib.syncbb_host_step.argtypes = [C.c_void_p, C.c_int64]
        lib.syncbb_host_init.argtypes = [C.c_void_p]
        inputs, state, scalars = syncbb_plan(layout_from_instance(inst), precision, "min", inst["var_rank"])
        k = dict(inputs, **host_state(state))
        d = _cabi.FgSyncbbDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        fill_desc(d, k, scalars)
        lib.syncbb_host_init(C.byref(d))
        t0 = time.perf_counter()
        lib.syncbb_host_step(C.byref(d), 1 << 62)
        dt = time.perf_counter() - t0
        return int(k["count"][0]) / dt


def main(argv=None):
    ap = argparse.ArgumentParser(prog="syncbb_throughput")
    ap.add_argument("--vars", type=int, default=29)
    ap.add_argument("--constraints", type=int, default=44)
    ap.add_argument("--seed", type=int, default=6)
    ap.add_argument("--precision", default="f64", choices=["f32", "f64"])
    ap.add_argument("--chunk", type=int, default=1 << 20, help="messages per launch")
    ap.add_argument("--host-steps", type=int, default=50000)
    args = ap.parse_args(argv)

    import torch
    if not torch.cuda.is_available():
        print("syncbb_throughput: no CUDA device (the SyncBB engine runs on the GPU only)", file=sys.stderr)
        return 2
    from _syncbb_oracle import SyncbbOracle
    from pydcop_b200.engine import SyncbbEngine
    from pydcop_b200.layout import layout_from_instance

    inst = instance(args.vars, args.constraints, args.seed)
    eng = SyncbbEngine(layout_from_instance(inst), precision=args.precision, var_rank=inst["var_rank"]).init()
    eng.step(1)                                   # first launch: module load
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    launches = 0
    while not eng.finished:                       # one host sync per launch of --chunk messages
        eng.step(args.chunk)
        launches += 1
    t1.record()
    t1.synchronize()
    ms = t0.elapsed_time(t1)
    steps, messages = eng.steps, eng.messages
    dev_rate = (steps - 1) / (ms * 1e-3)

    dt = np.float64 if args.precision == "f64" else np.float32
    o = SyncbbOracle(inst, dt, "min", inst["var_rank"]).init()
    h0 = time.perf_counter()
    o.run(args.host_steps)
    host_s = time.perf_counter() - h0
    host_rate = o.steps / host_s
    core_rate = one_core_rate(inst, args.precision)
    print(json.dumps({
        "workload": "syncbb_random_binary", "n_vars": args.vars, "n_constraints": args.constraints,
        "seed": args.seed, "precision": args.precision, "messages": messages, "steps": steps,
        "finished": eng.finished, "device": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(),
        "device_ms": round(ms, 1), "launches": launches + 1, "device_messages_per_s": round(dev_rate),
        "device_us_per_message": round(1e6 / dev_rate, 3),
        "host_oracle_steps": o.steps, "host_oracle_messages_per_s": round(host_rate),
        "device_over_host_oracle": round(dev_rate / host_rate, 1),
        "host_one_core_messages_per_s": round(core_rate) if core_rate else None,
        "device_over_host_one_core": round(dev_rate / core_rate, 3) if core_rate else None}))
    eng.close()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
