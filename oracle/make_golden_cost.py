#!/usr/bin/env python
"""Known answers of the UNMODIFIED reference's `solution_cost` (pydcop/dcop/dcop.py:319-367) for the
device reduction fg_solution_cost: random problems whose constraint tables AND variable costs contain
entries equal to `infinity` (hard constraints, counted, not summed), plus the reference's own
tests/instances/graph_coloring_10_4_15_0.1.yml (`10000 if vi == vj else 0`, `-i 10000`).

TEST INFRASTRUCTURE (build container only): writes tests/golden/solution_cost.json.

    python oracle/make_golden_cost.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402  (installs the import shims, imports the reference)
from pydcop.dcop.dcop import solution_cost  # noqa: E402
from pydcop.dcop.objects import Domain, VariableWithCostDict  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "solution_cost.json")


def arrays(variables, constraints):
    arr, _ = G.instance_arrays(variables, constraints)
    unary = [float(v.cost_for_val(x)) for v in variables for x in v.domain.values]
    return {"dom_size": arr["dom_size"].tolist(), "factor_ptr": arr["factor_ptr"].tolist(),
            "edge_var": arr["edge_var"].tolist(), "tables": [float(x) for x in arr["tables"]],
            "unary": unary}


def cases_for(variables, constraints, infinity, rng, n):
    out = []
    for _ in range(n):
        idx = [int(rng.integers(0, len(v.domain))) for v in variables]
        asg = {v.name: v.domain.values[i] for v, i in zip(variables, idx)}
        hard, soft = solution_cost(constraints, variables, asg, infinity)
        out.append({"value_index": idx, "violation": int(hard), "cost": float(soft)})
    return out


def main():
    rng = np.random.default_rng(7)
    problems = []
    for inf in (10000.0, 1e9, 777.0):
        dom = Domain("d", "", list(range(4)))
        variables = []
        for i in range(12):
            costs = {x: float(np.round(rng.uniform(0, 3), 3)) for x in range(4)}
            if i % 4 == 0:
                costs[int(rng.integers(0, 4))] = inf          # a forbidden value
            variables.append(VariableWithCostDict(f"v{i:02d}", dom, costs))
        constraints = []
        for j in range(20):
            a = (2, 2, 3, 1)[j % 4]
            scope = [variables[i] for i in rng.choice(12, size=a, replace=False)]
            m = np.round(rng.uniform(0, 9, size=(4,) * a), 2)
            if j % 3 == 0:
                m[rng.random(m.shape) < 0.35] = inf             # forbidden assignments
            constraints.append(NAryMatrixRelation(scope, m, name=f"c{j:02d}"))
        problems.append({"name": f"random_inf_{inf:g}", "infinity": inf, **arrays(variables, constraints),
                         "cases": cases_for(variables, constraints, inf, rng, 12)})
    dcop = load_dcop_from_file([os.path.join(G.ref_shim.INSTANCES,
                                             "graph_coloring_10_4_15_0.1.yml")])
    variables = list(dcop.variables.values())
    constraints = list(dcop.constraints.values())
    problems.append({"name": "graph_coloring_10_4_15_0.1", "infinity": 10000.0, **arrays(variables, constraints),
                     "cases": cases_for(variables, constraints, 10000.0, rng, 16)})
    json.dump(problems, open(OUT, "w"))
    print("wrote", OUT, [(p["name"], sum(c["violation"] for c in p["cases"])) for p in problems])


if __name__ == "__main__":
    main()
