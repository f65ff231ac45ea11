#!/usr/bin/env python
"""Generate tests/golden/mixeddsa_*.npz by running the UNMODIFIED reference MixedDSA in lock-step.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_mixeddsa.py [fixture names]

The reference module's build_computation forwards `stop_cycle`, which MixedDsaComputation.__init__ does not
accept, so the driver constructs `MixedDsaComputation(variable, constraints, variant=..., proba_hard=...,
proba_soft=..., mode=..., comp_def=...)` itself for every node of the constraints hypergraph, replaces
`message_sender` by a recorder and delivers the messages batch by batch, as oracle/make_golden.py does for DSA: one
batch is one round, in which every variable that has all its neighbours' values evaluates once (:272-373).

Constraints are given to the computations as NAryFunctionRelations over the tables: exists_violated_soft_constraint
calls `c(dict)` (:473), which only a function relation accepts (a matrix relation raises a ValueError).

Random draws are injected from oracle/philox.py: the start value (:233) with cycle 0xffffffff, the probability
tests and the choices of an evaluation with the computation's cycle_count (1 in round 1), u and the choice index
from the same block (oracle/make_golden.py _DsaRandom).

A variable without neighbours evaluates from on_start, with cycle_count 1, and never again.  Nobody sees its value,
so the fixture counts that evaluation as round 1: row 0 holds its start value.

Fixture keys: the constraint-hypergraph arrays of the GDBA fixtures (dom_size, factor_ptr, edge_var, table_off,
tables, var_ptr, var_con, unary, init_value) + per round k (row 0 = after on_start): value, cost (current_cost,
NaN while None), h_best (H of _compute_best_value, -1 without an evaluation) and branch (the case of :300-358 that
applied: 1 dH > 0, 2 soft improvement, 3 stuck with violated hard constraints, 4 stuck on a violated soft constraint,
5 none; 0 without an evaluation; + 8 when value_selection ran).
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import make_golden as G  # noqa: E402  (installs the reference shims)
import philox  # noqa: E402

from pydcop.algorithms import AlgorithmDef, ComputationDef  # noqa: E402
from pydcop.computations_graph import constraints_hypergraph  # noqa: E402
from pydcop.dcop.objects import Domain, Variable, VariableWithCostDict  # noqa: E402
from pydcop.dcop.relations import NAryFunctionRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
import pydcop.algorithms.mixeddsa as ref_mdsa  # noqa: E402

INF = float("inf")


class _MixedDsaRandom:
    """Replaces `random` in pydcop/algorithms/mixeddsa.py (stdlib; used :233, :301-334)."""

    @staticmethod
    def random():
        u, _ = philox.draw(G._Ctx.seed, G._Ctx.var, G._Ctx.comp.cycle_count)
        return u

    @staticmethod
    def choice(seq):
        c = G._Ctx.comp
        cycle = philox.INIT_CYCLE if c.cycle_count == 0 else c.cycle_count
        seq = list(seq)
        _, w = philox.draw(G._Ctx.seed, G._Ctx.var, cycle)
        return seq[philox.choice_index(w, len(seq))]


def table_relation(dims, table, name):
    """NAryFunctionRelation over a dense table (axis i <-> dims[i]); returns Python floats."""
    doms = [list(v.domain) for v in dims]
    m = np.asarray(table, dtype=np.float64)

    def f(**kw):
        return float(m[tuple(d.index(kw[v.name]) for v, d in zip(dims, doms))])
    return NAryFunctionRelation(f, dims, name=name)


def branch_of(comp, ev, mode, variant):
    """The case of :300-358 the evaluation recorded in `ev` took."""
    h_best, c_best, _ = ev["best"]
    dh = len(comp._violated_hard_cons) - h_best
    dc = comp._curr_dcop_cost - c_best
    if dh > 0:
        br = 1
    elif dh == 0 and ((mode == "min" and dc > 0) or (mode == "max" and dc < 0)):
        br = 2
    elif dh == 0 and dc == 0 and h_best > 0:
        br = 3
    elif dh == 0 and dc == 0 and ev.get("soft_violated") and variant in ("B", "C"):
        br = 4
    else:
        br = 5
    return br | (8 if ev.get("moved") else 0)


def run_mixeddsa(variables, constraints, params, mode, n_cycles, seed):
    variables, constraints = list(variables), list(constraints)
    p = dict(dict(proba_hard=0.7, proba_soft=0.5, variant="B"), **params)
    arr, vidx = G.instance_arrays(variables, constraints)
    V, N = len(variables), n_cycles
    g = constraints_hypergraph.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("mixeddsa", dict(p), mode=mode)
    comps, outbox, evals, start_value = {}, [], {}, {}

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    def hook(c):
        name = c.name
        best, soft, select = c._compute_best_value, c.exists_violated_soft_constraint, c.value_selection

        def compute_best_value():
            out = best()
            evals[name] = dict(best=(out[0], out[1], list(out[2])))
            return out

        def exists_violated_soft_constraint():
            out = soft()
            evals[name]["soft_violated"] = out
            return out

        def value_selection(val, cost=None):
            if name not in start_value:
                start_value[name] = val
            elif name in evals:
                evals[name]["moved"] = True
            return select(val, cost)
        c._compute_best_value = compute_best_value
        c.exists_violated_soft_constraint = exists_violated_soft_constraint
        c.value_selection = value_selection

    nodes = {}
    for node in g.nodes:
        c = ref_mdsa.MixedDsaComputation(node.variable, node.constraints, variant=p["variant"],
                                         proba_hard=p["proba_hard"], proba_soft=p["proba_soft"], mode=mode,
                                         comp_def=ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = lambda: None
        hook(c)
        comps[c.name] = c
        nodes[c.name] = node
    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for v in variables:
        for c in nodes[v.name].constraints:   # node.constraints order, the order MixedDsaComputation classifies in
            var_con.append(cidx[c.name])
        var_ptr.append(len(var_con))
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_con"] = np.array(var_con, dtype=np.int32)
    arr["unary"] = np.array([float(v.cost_for_val(x)) for v in variables for x in v.domain])
    doms = [list(v.domain) for v in variables]
    arr["init_value"] = np.array([doms[i].index(v.initial_value) if v.initial_value is not None else -1
                                  for i, v in enumerate(variables)], dtype=np.int32)

    rows = dict(cost=np.full((N + 1, V), np.nan), value=np.full((N + 1, V), -1, dtype=np.int32),
                h_best=np.full((N + 1, V), -1, dtype=np.int32), branch=np.zeros((N + 1, V), dtype=np.uint8))

    def snapshot(k):
        for i, v in enumerate(variables):
            c = comps[v.name]
            if k == 0:
                rows["value"][0, i] = doms[i].index(start_value[v.name])
                continue
            rows["value"][k, i] = doms[i].index(c.current_value)
            if c.current_cost is not None:
                rows["cost"][k, i] = c.current_cost
            if v.name in evals:
                rows["h_best"][k, i] = evals[v.name]["best"][0]
                rows["branch"][k, i] = branch_of(c, evals[v.name], mode, p["variant"])
        evals.clear()

    saved = ref_mdsa.random
    ref_mdsa.random = _MixedDsaRandom
    G._Ctx.seed = seed
    try:
        t0 = time.perf_counter()
        for v in variables:
            G._Ctx.var, G._Ctx.comp = vidx[v.name], comps[v.name]
            comps[v.name].start()
        start_evals = dict(evals)   # the variables without neighbours evaluated from on_start: round 1
        snapshot(0)
        evals.update(start_evals)
        for k in range(1, N + 1):
            batch, outbox[:] = list(outbox), []
            for s, d, m in batch:
                G._Ctx.var, G._Ctx.comp = vidx[d], comps[d]
                comps[d].on_message(s, m, 0)
            snapshot(k)
        dt = time.perf_counter() - t0
    finally:
        ref_mdsa.random = saved
    for i, v in enumerate(variables):   # a variable without neighbours evaluates once
        if not comps[v.name]._neighbors:
            assert comps[v.name].cycle_count == 2, (v.name, comps[v.name].cycle_count)
    arr.update(rows)
    meta = dict(algo="mixeddsa", mode=mode, params=dict(p, stop_cycle=0), n_cycles=N, seed=seed,
                ref_seconds=dt, ref_var_updates_per_s=V * N / dt if dt > 0 else 0.0)
    return arr, meta


def colouring(rng, n, dom, n_edges, hard_share, levels, arities=(2,), neg_inf=False, name="x"):
    """Hard `!=` colouring with soft preferences: a share of the constraints is hard (+inf, or -inf with neg_inf, on
    every entry whose scope variables are all equal; integer or dyadic costs elsewhere), the others soft; every third
    variable also gets a unary soft preference."""
    d = Domain(f"c{dom}", "", list(range(dom)))
    vs = [Variable(f"{name}{i:02d}", d) for i in range(n)]
    cs = []
    for j in range(n_edges):
        a = int(arities[j % len(arities)])
        scope = [vs[int(i)] for i in rng.choice(n, size=a, replace=False)]
        shape = (dom,) * a
        t = rng.integers(0, levels, size=shape).astype(float) / (8.0 if levels > 8 else 1.0)
        if rng.uniform() < hard_share:
            for x in range(dom):
                t[(x,) * a] = -INF if neg_inf else INF
        cs.append((scope, t, f"k{j:02d}"))
    for i in range(0, n, 3):
        cs.append(([vs[i]], rng.integers(0, levels, size=dom).astype(float), f"p{i:02d}"))
    return vs, cs


def with_extras(vs, cs):
    """Shapes every fixture holds: 'uno', whose only constraint is unary (it evaluates once, in round 1, through that
    constraint and its own cost), and 'iso', with a cost but no constraint (all its candidates cost 0)."""
    d3 = Domain("d3x", "", [0, 1, 2])
    uno = VariableWithCostDict("uno", d3, {0: 0.5, 1: 0.25, 2: 0.0})
    iso = VariableWithCostDict("iso", d3, {0: 0.5, 1: 0.25, 2: 0.25})
    return vs + [uno, iso], cs + [([uno], np.array([1.0, 1.0, 2.0]), "u_uno")]


def relations(cs):
    return [table_relation(scope, t, n) for scope, t, n in cs]


def with_costs(rng, vs, cs):
    out = [VariableWithCostDict(v.name, v.domain, {x: float(rng.integers(0, 9)) / 8.0 for x in v.domain}) for v in vs]
    by = {v.name: w for v, w in zip(vs, out)}
    return out, [([by[v.name] for v in scope], t, n) for scope, t, n in cs]


def with_initial(vs, cs):
    out = [Variable(v.name, v.domain, initial_value=(list(v.domain)[i % len(v.domain)] if i % 3 else None))
           for i, v in enumerate(vs)]
    by = {v.name: w for v, w in zip(vs, out)}
    return out, [([by[v.name] for v in scope], t, n) for scope, t, n in cs]


CASES = {
    # name: (params, mode, builder kwargs, transform)
    "mixeddsa_defaults": ({}, "min", dict(n=24, dom=3, n_edges=40, hard_share=0.6, levels=4), None),
    "mixeddsa_variant_A": ({"variant": "A"}, "min", dict(n=24, dom=3, n_edges=40, hard_share=0.6, levels=4), None),
    "mixeddsa_variant_C": ({"variant": "C"}, "min", dict(n=24, dom=3, n_edges=40, hard_share=0.6, levels=4), None),
    "mixeddsa_proba_1": ({"proba_hard": 1.0, "proba_soft": 1.0}, "min",
                         dict(n=24, dom=3, n_edges=44, hard_share=0.5, levels=3), None),
    "mixeddsa_proba_0": ({"proba_hard": 0.0, "proba_soft": 0.0}, "min",
                         dict(n=20, dom=3, n_edges=30, hard_share=0.5, levels=4), None),
    "mixeddsa_max_inf": ({}, "max", dict(n=24, dom=3, n_edges=40, hard_share=0.5, levels=5), None),
    "mixeddsa_neg_inf_min": ({"proba_soft": 0.8}, "min",
                             dict(n=22, dom=3, n_edges=36, hard_share=0.3, levels=4, neg_inf=True), None),
    "mixeddsa_neg_inf_max": ({}, "max", dict(n=22, dom=3, n_edges=36, hard_share=0.3, levels=4, neg_inf=True), None),
    "mixeddsa_nary": ({"proba_hard": 0.9}, "min",
                      dict(n=26, dom=3, n_edges=40, hard_share=0.4, levels=24, arities=(2, 3, 4, 1, 2)), None),
    "mixeddsa_var_costs": ({}, "min", dict(n=24, dom=4, n_edges=40, hard_share=0.5, levels=4), "costs"),
    "mixeddsa_initial_values": ({}, "min", dict(n=24, dom=3, n_edges=40, hard_share=0.6, levels=4), "initial"),
    "mixeddsa_stalemate": ({"proba_hard": 0.9}, "min", dict(n=12, dom=2, n_edges=40, hard_share=1.0, levels=1), None),
    "mixeddsa_ties": ({"proba_soft": 0.9}, "max", dict(n=24, dom=4, n_edges=36, hard_share=0.4, levels=2), None),
    "mixeddsa_rand_d12": ({}, "min", dict(n=24, dom=12, n_edges=60, hard_share=0.5, levels=10), None),
}


def main(only=(), out_dir=None):
    only = set(only)
    if out_dir:
        G.GOLDEN = out_dir

    def want(n):
        return not only or n in only

    for i, (name, (params, mode, kw, transform)) in enumerate(CASES.items()):
        if not want(name):
            continue
        rng = np.random.default_rng(90 if name.startswith(("mixeddsa_defaults", "mixeddsa_variant")) else 90 + i)
        vs, cs = colouring(rng, **kw)
        if transform == "costs":
            vs, cs = with_costs(rng, vs, cs)
        elif transform == "initial":
            vs, cs = with_initial(vs, cs)
        vs, cs = with_extras(vs, cs)
        arr, meta = run_mixeddsa(vs, relations(cs), params, mode, 14, seed=2468)
        G.save(name, arr, meta)
    if want("mixeddsa_ref_gc10"):
        dcop = load_dcop_from_file([os.path.join(G.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
        cs = [(list(c.dimensions), G.tabulate(c), c.name) for c in dcop.constraints.values()]
        vs, cs = with_extras(list(dcop.variables.values()), cs)
        arr, meta = run_mixeddsa(vs, relations(cs), {}, dcop.objective, 14, seed=11)
        G.save("mixeddsa_ref_gc10", arr, meta)


if __name__ == "__main__":
    main(sys.argv[1:])
