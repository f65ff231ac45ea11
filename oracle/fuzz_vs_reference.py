#!/usr/bin/env python
"""Random instances and parameters: the UNMODIFIED reference (lock-step, oracle/make_golden.py) against
the C oracle, cycle by cycle — extends the pinning beyond the committed fixtures.

TEST INFRASTRUCTURE (build container only).   python oracle/fuzz_vs_reference.py [n_cases] [seed]
Prints one JSON line: {"cases": n, "failures": [...]}.
"""
import json
import sys

import numpy as np

import os
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402
import make_golden_mgm as GM  # noqa: E402
import oracle as orc  # noqa: E402


def maxsum_case(rng):
    n_vars = int(rng.integers(4, 14))
    doms = [int(x) for x in rng.choice([2, 3, 4, 5], size=int(rng.integers(1, 3)))]
    arities = [int(a) for a in rng.choice([1, 2, 2, 3], size=3) if a <= n_vars]
    scale = float(rng.choice([1.0, 1e-6, 1e6, 1e18]))
    vs, cs = G.random_instance(rng, n_vars, doms, int(rng.integers(3, 16)), arities,
                               int_tables=bool(rng.integers(0, 2)), with_var_costs=bool(rng.integers(0, 2)),
                               n_unary=int(rng.integers(0, 3)))
    for c in cs:
        c._m[...] = c._m * scale
    params = {"damping": float(rng.choice([0.0, 0.3, 0.5, 0.9])),
              "damping_nodes": str(rng.choice(["vars", "factors", "both", "none"])),
              "stability": float(rng.choice([0.001, 0.1, 0.5])),
              "start_messages": str(rng.choice(["leafs", "leafs_vars", "all"])), "noise": 0.0}
    mode = str(rng.choice(["min", "max"]))
    hard = bool(rng.random() < 0.4)
    if hard:   # hard constraints: forbidden cells, and variables with every value forbidden
        inf = np.inf if mode == "min" else -np.inf
        for c in cs:
            if len(c.dimensions) > 1 and rng.random() < 0.5:
                c._m[rng.random(c._m.shape) < 0.3] = inf
        for j, i in enumerate(rng.choice(n_vars, size=int(rng.integers(1, 3)), replace=False)):
            cs.append(G.NAryMatrixRelation([vs[int(i)]], np.full(len(vs[int(i)].domain), inf), name=f"h{j:03d}"))
    arr, meta = G.run_maxsum(vs, cs, params, mode, 10, seed=int(rng.integers(1, 1000)))
    p = {k: v for k, v in params.items() if k != "noise"}
    o = orc.MaxSumOracle(arr, np.float64, mode=mode, **p).init()
    for k in range(11):
        if k:
            o.step()
        if not (np.array_equal(o.q, arr["q_state"][k], equal_nan=True) and np.array_equal(o.r, arr["r_state"][k], equal_nan=True)
                and np.array_equal(o.q_sent, arr["q_sent"][k]) and np.array_equal(o.r_sent, arr["r_sent"][k])):
            return f"maxsum messages differ at cycle {k}: {params} {mode} scale={scale} hard={hard}"
        if not np.array_equal(o.value, arr["value"][k]):
            # reported selection: ties at the ulp level are arrival-order dependent in the reference
            return None if scale != 1.0 else f"maxsum values differ at cycle {k}: {params} {mode} hard={hard}"
    return None


def dsa_case(rng):
    n_vars = int(rng.integers(5, 18))
    vs, cs = G.random_instance(rng, n_vars, [int(x) for x in rng.choice([2, 3, 4], size=2)], int(rng.integers(4, 20)),
                               [int(a) for a in rng.choice([2, 2, 3], size=2) if a <= n_vars])
    for c in cs:
        c._m[...] = rng.integers(0, 3, size=c._m.shape)
    params = {"variant": str(rng.choice(["A", "B", "C"])), "probability": float(rng.choice([0.3, 0.7, 1.0])),
              "stop_cycle": int(rng.choice([0, 0, 6]))}
    mode = str(rng.choice(["min", "max"]))
    seed = int(rng.integers(1, 1000))
    arr, meta = G.run_dsa(vs, cs, params, mode, 10, seed=seed)
    o = orc.DsaOracle(arr, np.float64, mode=mode, seed=seed, **params).init()
    for k in range(11):
        if k:
            o.step()
        if not np.array_equal(o.val, arr["value"][k]):
            return f"dsa values differ at cycle {k}: {params} {mode}"
    return None


def mgm_case(rng):
    n_vars = int(rng.integers(5, 18))
    vs, cs = G.random_instance(rng, n_vars, [int(x) for x in rng.choice([2, 3, 4], size=2)], int(rng.integers(4, 20)),
                               [int(a) for a in rng.choice([1, 2, 2, 3], size=3) if a <= n_vars])
    for c in cs:
        c._m[...] = rng.integers(0, 4, size=c._m.shape)
    if rng.integers(0, 2):
        vs2 = GM.dyadic_costs(rng, vs)
        cs, vs = GM.rebuild(cs, vs2), vs2
    params = {"stop_cycle": int(rng.choice([0, 0, 7]))}
    mode = str(rng.choice(["min", "max"]))
    seed = int(rng.integers(1, 1000))
    arr, meta = GM.run_mgm(vs, cs, params, mode, 9, seed=seed)
    o = orc.MgmOracle(arr, np.float64, mode=mode, seed=seed, **params).init()
    for k in range(10):
        if k:
            o.step()
        if not np.array_equal(o.val, arr["value"][k]):
            return f"mgm values differ at cycle {k}: {params} {mode}"
        known = ~np.isnan(arr["cost"][k])
        if not np.array_equal(o.cost[known], arr["cost"][k][known]):
            return f"mgm costs differ at cycle {k}: {params} {mode}"
    return None


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
    failures = []
    for i in range(n):
        f = (maxsum_case, dsa_case, mgm_case)[i % 3](rng)
        if f:
            failures.append(f"case {i}: {f}")
    print(json.dumps({"cases": n, "failures": failures}))


if __name__ == "__main__":
    main()
