#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference in deterministic lock-step.

TEST INFRASTRUCTURE (build container only: needs /root/reference).  Run:
    python oracle/make_golden.py            # regenerates every fixture

What it does (SURVEY.md §8c, Appendix B): instantiates the reference's own
`MaxSumFactorComputation` / `MaxSumVariableComputation` (pydcop/algorithms/maxsum.py:279,450)
and `DsaComputation` (pydcop/algorithms/dsa.py:214) through the reference's
`build_computation(ComputationDef(node, algo))` (pydcop/infrastructure/computations.py:1156),
replaces `message_sender` by a recorder, and delivers all messages round by round.  One delivery
round == one synchronous cycle (pydcop/infrastructure/computations.py:633-642).

Each fixture holds the instance as flat arrays (the same arrays the engine's array front door
takes) and the full per-cycle trajectory: receiver-side message state, send flags, selected
values and costs.  DSA's random draws are injected from oracle/philox.py.
"""
import json
import os
import random as _stdlib_random
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.install()
import logging  # noqa: E402
logging.disable(logging.CRITICAL)
import philox  # noqa: E402

from pydcop.algorithms import AlgorithmDef, ComputationDef  # noqa: E402
from pydcop.computations_graph import constraints_hypergraph, factor_graph  # noqa: E402
from pydcop.dcop.objects import Domain, Variable, VariableWithCostDict  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402
import pydcop.algorithms.dsa as ref_dsa  # noqa: E402
import pydcop.infrastructure.computations as ref_computations  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
INSTANCES = ref_shim.INSTANCES


# --------------------------------------------------------------------------------------
# instance -> flat arrays
# --------------------------------------------------------------------------------------
def tabulate(constraint):
    """Dense row-major table of a reference Constraint, axis i <-> dimensions[i]
    (layout of NAryMatrixRelation._m, pydcop/dcop/relations.py:716-733)."""
    dims = constraint.dimensions
    shape = tuple(len(v.domain) for v in dims)
    t = np.zeros(shape, dtype=np.float64)
    for idx in np.ndindex(*shape):
        asg = {v.name: v.domain.values[i] if hasattr(v.domain, "values") else list(v.domain)[i]
               for v, i in zip(dims, idx)}
        t[idx] = constraint(**asg)
    return t


def instance_arrays(variables, constraints):
    variables = list(variables)
    constraints = list(constraints)
    vidx = {v.name: i for i, v in enumerate(variables)}
    dom_size = np.array([len(v.domain) for v in variables], dtype=np.int32)
    factor_ptr = [0]
    edge_var = []
    table_off = [0]
    tables = []
    for c in constraints:
        for v in c.dimensions:
            edge_var.append(vidx[v.name])
        factor_ptr.append(len(edge_var))
        t = tabulate(c).reshape(-1)
        tables.append(t)
        table_off.append(table_off[-1] + t.size)
    arr = dict(
        dom_size=dom_size,
        factor_ptr=np.array(factor_ptr, dtype=np.int32),
        edge_var=np.array(edge_var, dtype=np.int32),
        table_off=np.array(table_off, dtype=np.int64),
        tables=np.concatenate(tables) if tables else np.zeros(0),
    )
    arr["var_names"] = np.array([v.name for v in variables])
    arr["factor_names"] = np.array([c.name for c in constraints])
    return arr, vidx


def edge_offsets(arr):
    d = arr["dom_size"][arr["edge_var"]]
    off = np.zeros(len(d) + 1, dtype=np.int64)
    np.cumsum(d, out=off[1:])
    return off


# --------------------------------------------------------------------------------------
# MaxSum lock-step
# --------------------------------------------------------------------------------------
def run_maxsum(variables, constraints, params, mode, n_cycles, seed):
    variables = list(variables)
    constraints = list(constraints)
    _stdlib_random.seed(seed)  # noise draw, pydcop/dcop/objects.py:566-567
    arr, vidx = instance_arrays(variables, constraints)
    V, F = len(variables), len(constraints)
    E = len(arr["edge_var"])
    moff = edge_offsets(arr)
    M = int(moff[-1])
    fidx = {c.name: i for i, c in enumerate(constraints)}
    # edge id of (factor, variable)
    edge_of = {}
    for f, c in enumerate(constraints):
        for j, v in enumerate(c.dimensions):
            edge_of[(c.name, v.name)] = arr["factor_ptr"][f] + j

    g = factor_graph.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("maxsum", dict(params), mode=mode)
    comps, outbox = {}, []

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        comps[c.name] = c

    # variable-side CSR in `links` order (maxsum.py:466) and the unary costs the
    # computations really use (incl. noise, maxsum.py:477-487)
    var_ptr = [0]
    var_edge = []
    unary = []
    init_value = np.full(V, -1, dtype=np.int32)
    for v in variables:
        comp = comps[v.name]
        for fname in comp.factors:
            var_edge.append(edge_of[(fname, v.name)])
        var_ptr.append(len(var_edge))
        vv = comp._variable
        dom = list(v.domain)
        unary.extend(float(vv.cost_for_val(x)) for x in dom)
        if v.initial_value is not None:
            init_value[vidx[v.name]] = dom.index(v.initial_value)
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_edge"] = np.array(var_edge, dtype=np.int32)
    arr["unary"] = np.array(unary, dtype=np.float64)
    arr["init_value"] = init_value

    N = n_cycles
    r_state = np.zeros((N + 1, M))
    q_state = np.zeros((N + 1, M))
    r_valid = np.zeros((N + 1, E), dtype=bool)
    q_valid = np.zeros((N + 1, E), dtype=bool)
    r_sent = np.zeros((N + 1, E), dtype=bool)
    q_sent = np.zeros((N + 1, E), dtype=bool)
    value = np.zeros((N + 1, V), dtype=np.int32)
    value_cost = np.zeros((N + 1, V))
    doms = [list(v.domain) for v in variables]

    def record(k):
        if k > 0:
            r_state[k], q_state[k] = r_state[k - 1], q_state[k - 1]
            r_valid[k], q_valid[k] = r_valid[k - 1], q_valid[k - 1]
        for s, d, m in outbox:
            if m.type != "max_sum":
                continue
            if s in fidx:  # factor -> variable
                e = edge_of[(s, d)]
                dom = doms[vidx[d]]
                r_state[k, moff[e]:moff[e + 1]] = [m.costs[x] for x in dom]
                r_valid[k, e] = True
                r_sent[k, e] = True
            else:
                e = edge_of[(d, s)]
                dom = doms[vidx[s]]
                q_state[k, moff[e]:moff[e + 1]] = [m.costs[x] for x in dom]
                q_valid[k, e] = True
                q_sent[k, e] = True
        for i, v in enumerate(variables):
            c = comps[v.name]
            value[k, i] = doms[i].index(c.current_value)
            value_cost[k, i] = c.current_cost if c.current_cost is not None else np.nan

    t0 = time.perf_counter()
    for c in comps.values():
        c.start()  # cycle 0
    record(0)
    for k in range(1, N + 1):
        batch, outbox[:] = list(outbox), []
        for s, d, m in batch:
            comps[d].on_message(s, m, 0)
        record(k)
    dt = time.perf_counter() - t0

    arr.update(r_state=r_state, q_state=q_state, r_valid=r_valid, q_valid=q_valid,
               r_sent=r_sent, q_sent=q_sent, value=value, value_cost=value_cost)
    meta = dict(algo="maxsum", mode=mode, params=dict(algo.params), n_cycles=N, seed=seed,
                ref_seconds=dt, ref_updates_per_s=2 * E * N / dt if dt > 0 else 0.0)
    return arr, meta


# --------------------------------------------------------------------------------------
# DSA lock-step with injected draws
# --------------------------------------------------------------------------------------
class _Ctx:
    seed = 0
    var = 0
    comp = None


class _DsaRandom:
    """Replaces `random` in pydcop/algorithms/dsa.py (stdlib; :96, used :411-412)."""

    @staticmethod
    def random():
        u, _ = philox.draw(_Ctx.seed, _Ctx.var, _Ctx.comp.cycle_count)
        return u

    @staticmethod
    def choice(seq):
        _, w = philox.draw(_Ctx.seed, _Ctx.var, _Ctx.comp.cycle_count)
        return seq[philox.choice_index(w, len(seq))]


class _InitRandom:
    """Replaces numpy `random` in pydcop/infrastructure/computations.py (:45, used :1086)."""

    @staticmethod
    def choice(seq):
        seq = list(seq)
        _, w = philox.draw(_Ctx.seed, _Ctx.var, philox.INIT_CYCLE)
        return seq[philox.choice_index(w, len(seq))]


def run_dsa(variables, constraints, params, mode, n_cycles, seed):
    variables = list(variables)
    constraints = list(constraints)
    arr, vidx = instance_arrays(variables, constraints)
    V = len(variables)
    g = constraints_hypergraph.build_computation_graph(
        None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("dsa", dict(params), mode=mode)
    comps, outbox = {}, []
    finished = set()

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = (lambda name=c.name: finished.add(name))
        comps[c.name] = c
    for v in variables:
        for c in comps[v.name].constraints:  # node.constraints order, dsa.py:255
            var_con.append(cidx[c.name])
        var_ptr.append(len(var_con))
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_con"] = np.array(var_con, dtype=np.int32)
    # variable costs are NOT used by DSA's decision (dead branch relations.py:1630) but an
    # isolated variable picks argopt of its own cost (dsa.py:278-289)
    arr["unary"] = np.array([float(v.cost_for_val(x)) for v in variables for x in v.domain])

    saved = ref_dsa.random, ref_computations.random
    ref_dsa.random, ref_computations.random = _DsaRandom, _InitRandom
    _Ctx.seed = seed
    N = n_cycles
    doms = [list(v.domain) for v in variables]
    value = np.zeros((N + 1, V), dtype=np.int32)
    cycle_count = np.zeros((N + 1, V), dtype=np.int32)

    def record(k):
        for i, v in enumerate(variables):
            value[k, i] = doms[i].index(comps[v.name].current_value)
            cycle_count[k, i] = comps[v.name].cycle_count

    try:
        t0 = time.perf_counter()
        for v in variables:
            _Ctx.var, _Ctx.comp = vidx[v.name], comps[v.name]
            comps[v.name].start()
        record(0)
        for k in range(1, N + 1):
            batch, outbox[:] = list(outbox), []
            for s, d, m in batch:
                _Ctx.var, _Ctx.comp = vidx[d], comps[d]
                comps[d].on_message(s, m, 0)
            record(k)
        dt = time.perf_counter() - t0
    finally:
        ref_dsa.random, ref_computations.random = saved
    arr.update(value=value, cycle_count=cycle_count)
    arr["finished"] = np.array([v.name in finished for v in variables])
    meta = dict(algo="dsa", mode=mode, params=dict(algo.params), n_cycles=N, seed=seed,
                ref_seconds=dt, ref_var_updates_per_s=V * N / dt if dt > 0 else 0.0)
    return arr, meta


# --------------------------------------------------------------------------------------
# instance builders (reference classes only)
# --------------------------------------------------------------------------------------
def random_instance(rng, n_vars, dom_sizes, n_factors, arities, int_tables=True,
                    with_var_costs=False, n_unary=0, name="i"):
    """Random factor graph: each factor draws `arity` distinct variables uniformly;
    tables are integers(0,10) like the soft graph-colouring generator
    (pydcop/commands/generators/graphcoloring.py:370) or uniform floats."""
    doms = {}
    variables = []
    for i in range(n_vars):
        d = int(dom_sizes[i % len(dom_sizes)])
        if d not in doms:
            doms[d] = Domain(f"d{d}", "", list(range(d)))
        if with_var_costs:
            costs = {x: float(np.round(rng.uniform(0, 1), 3)) for x in range(d)}
            variables.append(VariableWithCostDict(f"v{i:03d}", doms[d], costs))
        else:
            variables.append(Variable(f"v{i:03d}", doms[d]))
    constraints = []
    for j in range(n_factors):
        a = int(arities[j % len(arities)])
        scope_idx = rng.choice(n_vars, size=a, replace=False)
        scope = [variables[i] for i in scope_idx]
        shape = tuple(len(v.domain) for v in scope)
        if int_tables:
            m = rng.integers(0, 10, size=shape).astype(np.float64)
        else:
            m = np.round(rng.uniform(-5, 5, size=shape), 4)
        constraints.append(NAryMatrixRelation(scope, m, name=f"c{j:03d}"))
    for j in range(n_unary):
        v = variables[int(rng.integers(0, n_vars))]
        m = np.round(rng.uniform(0, 2, size=(len(v.domain),)), 4)
        constraints.append(NAryMatrixRelation([v], m, name=f"u{j:03d}"))
    return variables, constraints


def ising_instance(rng, rows, cols):
    """Toroidal Ising grid restating pydcop/commands/generators/ising.py:274-331,362-420:
    d=2, binary table [[k,-k],[-k,k]], k~U(-1.6,1.6); unary factor [u,-u], u~U(-0.05,0.05)."""
    dom = Domain("spin", "", [0, 1])
    variables = [Variable(f"v_{r}_{c}", dom) for r in range(rows) for c in range(cols)]
    constraints = []
    for r in range(rows):
        for c in range(cols):
            v = variables[r * cols + c]
            for (r2, c2) in (((r + 1) % rows, c), (r, (c + 1) % cols)):
                w = variables[r2 * cols + c2]
                if w is v:
                    continue
                k = rng.uniform(-1.6, 1.6)
                constraints.append(NAryMatrixRelation(
                    [v, w], np.array([[k, -k], [-k, k]]), name=f"cb_{r}_{c}_{r2}_{c2}"))
    for r in range(rows):
        for c in range(cols):
            u = rng.uniform(-0.05, 0.05)
            constraints.append(NAryMatrixRelation(
                [variables[r * cols + c]], np.array([u, -u]), name=f"cu_{r}_{c}"))
    return variables, constraints


def tree_instance(rng, n_vars, d):
    """Random tree (so `leafs` start messages matter) + one isolated variable with initial_value."""
    dom = Domain("d", "", list(range(d)))
    variables = [Variable(f"t{i:02d}", dom) for i in range(n_vars)]
    constraints = []
    for i in range(1, n_vars):
        p = int(rng.integers(0, i))
        m = rng.integers(0, 10, size=(d, d)).astype(np.float64)
        constraints.append(NAryMatrixRelation([variables[p], variables[i]], m, name=f"e{i:02d}"))
    variables.append(Variable("iso", dom, initial_value=d - 1))
    return variables, constraints


def save(name, arr, meta):
    os.makedirs(GOLDEN, exist_ok=True)
    path = os.path.join(GOLDEN, name + ".npz")
    np.savez_compressed(path, meta=np.array(json.dumps(meta)), **arr)
    kind = meta["algo"]
    rate = meta.get("ref_updates_per_s", meta.get("ref_var_updates_per_s", 0.0))
    print(f"{name:32s} {kind:6s} {os.path.getsize(path) / 1024:8.1f} KiB  "
          f"ref {meta['ref_seconds']:.2f}s  {rate:10.0f} upd/s")


def main():
    only = set(sys.argv[1:])

    def want(n):
        return not only or n in only

    # ---- MaxSum -------------------------------------------------------------------
    if want("ms_gc10_default"):
        # BASELINE config C1: graph_coloring 10 vars / 3 colours, default params
        dcop = load_dcop_from_file([os.path.join(INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
        arr, meta = run_maxsum(dcop.variables.values(), dcop.constraints.values(),
                               {}, dcop.objective, 40, seed=1)
        save("ms_gc10_default", arr, meta)
    if want("ms_gc3_costs"):
        dcop = load_dcop_from_file([os.path.join(INSTANCES, "graph_coloring1.yaml")])
        arr, meta = run_maxsum(dcop.variables.values(), dcop.constraints.values(),
                               {}, dcop.objective, 30, seed=2)
        save("ms_gc3_costs", arr, meta)
    if want("ms_secp_simple1"):
        dcop = load_dcop_from_file([os.path.join(INSTANCES, "secp_simple1.yaml")])
        arr, meta = run_maxsum(dcop.variables.values(), dcop.constraints.values(),
                               {}, dcop.objective, 30, seed=3)
        save("ms_secp_simple1", arr, meta)
    if want("ms_rand_bin_d10"):
        rng = np.random.default_rng(10)
        vs, cs = random_instance(rng, 30, [10], 60, [2])
        arr, meta = run_maxsum(vs, cs, {}, "min", 25, seed=4)
        save("ms_rand_bin_d10", arr, meta)
    if want("ms_rand_mixed"):
        rng = np.random.default_rng(11)
        vs, cs = random_instance(rng, 24, [2, 3, 5, 4], 30, [2, 2, 3, 1], int_tables=False,
                                 with_var_costs=True, n_unary=4)
        arr, meta = run_maxsum(vs, cs, {"noise": 0.0}, "min", 30, seed=5)
        save("ms_rand_mixed", arr, meta)
    if want("ms_arity3_d4"):
        rng = np.random.default_rng(12)
        vs, cs = random_instance(rng, 18, [4], 16, [3])
        arr, meta = run_maxsum(vs, cs, {}, "min", 25, seed=6)
        save("ms_arity3_d4", arr, meta)
    if want("ms_arity4_mixed"):
        rng = np.random.default_rng(13)
        vs, cs = random_instance(rng, 12, [3, 2, 4], 8, [4, 3, 2], int_tables=False)
        arr, meta = run_maxsum(vs, cs, {}, "min", 20, seed=7)
        save("ms_arity4_mixed", arr, meta)
    if want("ms_ising_4x4"):
        rng = np.random.default_rng(14)
        vs, cs = ising_instance(rng, 4, 4)
        arr, meta = run_maxsum(vs, cs, {}, "min", 30, seed=8)
        save("ms_ising_4x4", arr, meta)
    if want("ms_tree_leafs"):
        rng = np.random.default_rng(15)
        vs, cs = tree_instance(rng, 14, 4)
        arr, meta = run_maxsum(vs, cs, {}, "min", 30, seed=9)
        save("ms_tree_leafs", arr, meta)
    # parameter sweeps on one small instance
    sweeps = {
        "ms_p_nodamp": ({"damping_nodes": "none"}, "min"),
        "ms_p_damp_vars": ({"damping_nodes": "vars", "damping": 0.8}, "min"),
        "ms_p_damp_factors": ({"damping_nodes": "factors", "damping": 0.3}, "min"),
        "ms_p_stab_tight": ({"stability": 0.001}, "min"),
        "ms_p_stab_loose": ({"stability": 0.5}, "min"),
        "ms_p_start_leafs_vars": ({"start_messages": "leafs_vars"}, "min"),
        "ms_p_start_all": ({"start_messages": "all"}, "min"),
        "ms_p_max_mode": ({}, "max"),
        "ms_p_noise0_int": ({"noise": 0.0}, "min"),
    }
    for name, (params, mode) in sweeps.items():
        if want(name):
            rng = np.random.default_rng(20)
            vs, cs = random_instance(rng, 16, [4, 3], 22, [2, 2, 3, 1])
            arr, meta = run_maxsum(vs, cs, params, mode, 25, seed=21)
            save(name, arr, meta)

    # ---- DSA ------------------------------------------------------------------------
    dsa_cases = {
        "dsa_B_default": ({"stop_cycle": 0}, "min", [2]),
        "dsa_A": ({"variant": "A"}, "min", [2]),
        "dsa_C": ({"variant": "C", "probability": 0.5}, "min", [2]),
        "dsa_B_max": ({"variant": "B"}, "max", [2]),
        "dsa_B_arity_pmode": ({"p_mode": "arity"}, "min", [2, 3]),
        "dsa_B_ternary": ({"probability": 0.6}, "min", [3, 2, 2]),
        "dsa_B_stop10": ({"stop_cycle": 10}, "min", [2]),
    }
    for name, (params, mode, arities) in dsa_cases.items():
        if want(name):
            rng = np.random.default_rng(30)
            # few distinct integer costs => many ties => exercises the delta==0 branches
            vs, cs = random_instance(rng, 30, [5, 4], 45, arities)
            for c in cs:
                c._m[...] = rng.integers(0, 3, size=c._m.shape)
            if params.get("p_mode") != "arity":
                # (p_mode=arity divides by zero for an isolated variable, dsa.py:258-260)
                vs.append(Variable("iso", Domain("diso", "", [0, 1, 2])))
            arr, meta = run_dsa(vs, cs, params, mode, 30, seed=1234)
            save(name, arr, meta)
    if want("dsa_gc10"):
        dcop = load_dcop_from_file([os.path.join(INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
        arr, meta = run_dsa(dcop.variables.values(), dcop.constraints.values(),
                            {}, dcop.objective, 30, seed=77)
        save("dsa_gc10", arr, meta)
    if want("dsa_rand_d20"):
        rng = np.random.default_rng(31)
        vs, cs = random_instance(rng, 40, [20], 120, [2])
        arr, meta = run_dsa(vs, cs, {}, "min", 20, seed=5)
        save("dsa_rand_d20", arr, meta)


if __name__ == "__main__":
    main()
