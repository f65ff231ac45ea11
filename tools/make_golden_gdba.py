#!/usr/bin/env python
"""Generate tests/golden/gdba_*.npz by running the UNMODIFIED reference GDBA in lock-step.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_gdba.py [fixture names]

Same method as oracle/make_golden_mgm.py: the reference's own `GdbaComputation`
(pydcop/algorithms/gdba.py:189) is built through `build_computation(ComputationDef(node, algo))`,
`message_sender` is replaced by a recorder and the messages are delivered batch by batch.  One round
is TWO batches: every ok message (each variable then evaluates its values and posts its improve,
gdba.py:352-387), then every improve message (each variable then moves or breaks out and posts its
value for the next round, :493-541).  A variable that finishes a round early posts its next ok
messages into the next batch, so nobody sees a value of the next round early.  The reference has
no stop_cycle: the driver stops delivering after n_cycles rounds.

Random draws (:319 start value, :376 pick among the best values) are injected from
oracle/philox.py, keyed (seed; variable, cycle) as MGM's are.

Fixture keys: the constraint-hypergraph arrays of the MGM fixtures (dom_size, factor_ptr, edge_var,
table_off, tables, var_ptr, var_con, unary, init_value, var_rank) + per round k (row 0 = after
on_start): value, cost (the reference's current_cost at the end of the round, NaN while None),
improve (_my_improve), new_value, violated (per variable and slot in var_con order: the constraint
is in _violated_constraints), breakout (the round increased at least one modifier) and modifiers
(per variable, slot and table entry: the modifier a read sees, `dict.get(key, base)` on the
reference's defaultdict so that recording inserts nothing).
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
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402
import pydcop.algorithms.gdba as ref_gdba  # noqa: E402


class _GdbaRandom:
    """Replaces `random` in pydcop/algorithms/gdba.py (stdlib; used :319, :376)."""

    @staticmethod
    def choice(seq):
        c = G._Ctx.comp
        cycle = philox.INIT_CYCLE if c._waiting_mode == "starting" else c.cycle_count
        seq = list(seq)
        _, w = philox.draw(G._Ctx.seed, G._Ctx.var, cycle)
        return seq[philox.choice_index(w, len(seq))]


def read_modifiers(comp):
    """Every modifier of `comp` as _get_modifier_for_assignment reads it, per slot and table entry."""
    base = 0 if comp._modifier_mode == "A" else 1
    out = []
    for rel, _, _ in comp.__constraints__:
        mods = comp.__constraints_modifiers__[rel]
        dims = rel.dimensions
        doms = [list(v.domain) for v in dims]
        for idx in np.ndindex(*[len(d) for d in doms]):
            key = frozenset({v.name: d[i] for v, d, i in zip(dims, doms, idx)}.items())
            out.append(mods.get(key, base))
    return out


def run_gdba(variables, constraints, params, mode, n_cycles, seed):
    variables, constraints = list(variables), list(constraints)
    arr, vidx = G.instance_arrays(variables, constraints)
    V, N = len(variables), n_cycles
    g = constraints_hypergraph.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("gdba", dict(params), mode=mode)
    comps, outbox = {}, []

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    nodes = {}
    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = lambda: None
        comps[c.name] = c
        nodes[c.name] = node
    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for v in variables:
        comp = comps[v.name]
        for (rel, _, _), c in zip(comp.__constraints__, nodes[v.name].constraints):   # gdba.py:252
            assert [d.name for d in rel.dimensions] == [d.name for d in c.dimensions]
            var_con.append(cidx[c.name])
        var_ptr.append(len(var_con))
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_con"] = np.array(var_con, dtype=np.int32)
    arr["unary"] = np.array([float(v.cost_for_val(x)) for v in variables for x in v.domain])
    doms = [list(v.domain) for v in variables]
    arr["init_value"] = np.array([doms[i].index(v.initial_value) if v.initial_value is not None else -1
                                  for i, v in enumerate(variables)], dtype=np.int32)
    order = sorted(range(V), key=lambda i: variables[i].name)
    rank = np.zeros(V, dtype=np.int32)
    rank[order] = np.arange(V, dtype=np.int32)
    arr["var_rank"] = rank
    S = len(var_con)

    rows = {k: np.full((N + 1, V), np.nan) for k in ("cost", "improve")}
    rows["value"] = np.full((N + 1, V), -1, dtype=np.int32)
    rows["new_value"] = np.full((N + 1, V), -1, dtype=np.int32)
    rows["breakout"] = np.zeros((N + 1, V), dtype=np.uint8)
    rows["violated"] = np.zeros((N + 1, S), dtype=np.uint8)
    mods = []

    increased = set()
    orig_increase = ref_gdba.GdbaComputation._increase_cost

    def increase_wrapper(self, constraint):
        increased.add(self.name)
        return orig_increase(self, constraint)

    def snapshot(k):
        for i, v in enumerate(variables):
            c = comps[v.name]
            rows["value"][k, i] = doms[i].index(c.current_value)
            if c.current_cost is not None:
                rows["cost"][k, i] = c.current_cost
            rows["breakout"][k, i] = v.name in increased
        mods.append(np.array([m for v in variables for m in read_modifiers(comps[v.name])], dtype=np.int32))

    def deliver():
        batch, outbox[:] = list(outbox), []
        for s, d, m in batch:
            G._Ctx.var, G._Ctx.comp = vidx[d], comps[d]
            comps[d].on_message(s, m, 0)

    saved = ref_gdba.random
    ref_gdba.random = _GdbaRandom
    ref_gdba.GdbaComputation._increase_cost = increase_wrapper
    G._Ctx.seed = seed
    try:
        t0 = time.perf_counter()
        for v in variables:
            G._Ctx.var, G._Ctx.comp = vidx[v.name], comps[v.name]
            comps[v.name].start()
        snapshot(0)
        for k in range(1, N + 1):
            deliver()                      # ok messages of round k
            for i, v in enumerate(variables):
                c = comps[v.name]
                if not c.neighbors:
                    continue
                rows["improve"][k, i] = c._my_improve
                rows["new_value"][k, i] = doms[i].index(c._new_value)
                for s in range(var_ptr[i], var_ptr[i + 1]):
                    rel = c.__constraints__[s - var_ptr[i]][0]
                    rows["violated"][k, s] = any(r is rel for r in c._violated_constraints)
            increased.clear()
            deliver()                      # improve messages of round k
            snapshot(k)
        dt = time.perf_counter() - t0
    finally:
        ref_gdba.random = saved
        ref_gdba.GdbaComputation._increase_cost = orig_increase
    arr.update(rows)
    arr["modifiers"] = np.stack(mods)
    meta = dict(algo="gdba", mode=mode, params=dict(algo.params, stop_cycle=0), n_cycles=N, seed=seed,
                ref_seconds=dt, ref_var_updates_per_s=V * N / dt if dt > 0 else 0.0)
    return arr, meta


def rebuild(constraints, variables):
    by_name = {v.name: v for v in variables}
    return [NAryMatrixRelation([by_name[v.name] for v in c.dimensions], c._m, name=c.name)
            for c in constraints]


def with_extras(vs, cs, rng, levels):
    """The shapes every GDBA fixture contains, attached to the instance's first variable v0:
      - a ternary constraint t(s0, s1, s2) where s0 has no other constraint, so it spans s0's
        neighbourhood (E / R / C writes land on it);
      - s1 also constrained with v0 (its ternary constraint does not span: E / R / C change nothing);
      - a degree-1 variable 'leaf' with a binary constraint to s2 (spans) and a unary one (does not);
      - 'uno', whose only constraint is unary, and 'iso' without any constraint (own costs only)."""
    d3 = Domain("d3x", "", [0, 1, 2])
    by_name = {v.name: v for v in vs}
    v0 = vs[0]
    cost_like = type(v0) is VariableWithCostDict
    mk = (lambda n: VariableWithCostDict(n, d3, {0: 0.25, 1: 0.0, 2: 0.5})) if cost_like else \
        (lambda n: Variable(n, d3))
    s0, s1, s2, leaf = mk("s0"), mk("s1"), mk("s2"), mk("w_leaf")
    uno = Variable("uno", d3)
    iso = VariableWithCostDict("iso", d3, {0: 0.5, 1: 0.25, 2: 0.25})

    def table(*shape):
        return (rng.integers(0, levels, size=shape).astype(float) if levels
                else np.round(rng.uniform(-3, 7, size=shape), 3))
    # stuck on a maximal entry of a spanning constraint (violated under NZ, NM and MX): s0 whenever
    # s1 = 0, and the leaf, which its unary cost keeps at 0
    top = float(levels - 1) if levels else 7.0
    t_s, b_leaf = table(3, 3, 3), table(3, 3)
    t_s[:, 0, :] = top
    b_leaf[0, :] = top
    cs = cs + [NAryMatrixRelation([s0, s1, s2], t_s, name="t_s"),
               NAryMatrixRelation([s1, by_name[v0.name]], table(3, len(v0.domain)), name="b_s1"),
               NAryMatrixRelation([leaf, s2], b_leaf, name="b_leaf"),
               NAryMatrixRelation([leaf], np.array([0.0, 3 * top + 3, 3 * top + 3]), name="u_leaf"),
               NAryMatrixRelation([uno], np.array([2.0, 1.0, 1.0]), name="u_uno")]
    return vs + [s0, s1, s2, leaf, uno, iso], cs


GRID = [(m, vi, inc) for m in ("A", "M") for vi in ("NZ", "NM", "MX") for inc in ("E", "R", "C", "T")]
CASES = {
    # name: (params, mode, arities, cost levels (0 = non-dyadic floats), var costs, initial values)
    **{f"gdba_{m}_{vi}_{inc}": ({"modifier": m, "violation": vi, "increase_mode": inc}, "min", [2, 2, 3], 4,
                                False, False) for m, vi, inc in GRID},
    "gdba_max_A_NZ_E": ({"modifier": "A", "violation": "NZ", "increase_mode": "E"}, "max", [2, 2, 3], 4, False, False),
    "gdba_max_M_MX_T": ({"modifier": "M", "violation": "MX", "increase_mode": "T"}, "max", [2, 3], 3, False, False),
    "gdba_var_costs": ({"increase_mode": "T"}, "min", [2, 2, 3], 4, True, False),
    "gdba_initial_values": ({"increase_mode": "C"}, "min", [2, 2, 3], 4, False, True),
    "gdba_float": ({"modifier": "M", "violation": "NM", "increase_mode": "R"}, "min", [2, 3], 0, False, False),
}


def main(only=(), out_dir=None):
    only = set(only)
    if out_dir:
        G.GOLDEN = out_dir

    def want(n):
        return not only or n in only

    for name, (params, mode, arities, levels, var_costs, init) in CASES.items():
        if not want(name):
            continue
        rng = np.random.default_rng(70)
        vs, cs = G.random_instance(rng, 22, [4, 3, 2], 26, arities)
        for c in cs:
            c._m[...] = (rng.integers(0, levels, size=c._m.shape) if levels
                         else np.round(rng.uniform(-3, 7, size=c._m.shape), 3))
        if init:
            vs2 = [Variable(v.name, v.domain, initial_value=(list(v.domain)[i % len(v.domain)] if i % 3 else None))
                   for i, v in enumerate(vs)]
            cs, vs = rebuild(cs, vs2), vs2
        if var_costs:
            vs2 = [VariableWithCostDict(v.name, v.domain, {x: float(rng.integers(0, 9)) / 4.0 for x in v.domain})
                   for v in vs]
            cs, vs = rebuild(cs, vs2), vs2
        vs, cs = with_extras(vs, cs, rng, levels)
        arr, meta = run_gdba(vs, cs, params, mode, 14, seed=1357)
        G.save(name, arr, meta)
    if want("gdba_gc10"):
        dcop = load_dcop_from_file([os.path.join(G.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
        # as matrices: the reference converts function relations with ndarray.itemset, gone in NumPy 2
        cs = [NAryMatrixRelation(c.dimensions, G.tabulate(c), name=c.name) for c in dcop.constraints.values()]
        vs, cs = with_extras(list(dcop.variables.values()), cs, np.random.default_rng(71), 3)
        arr, meta = run_gdba(vs, cs, {"violation": "NM"}, dcop.objective, 14, seed=93)
        G.save("gdba_gc10", arr, meta)
    if want("gdba_rand_d12"):
        rng = np.random.default_rng(72)
        vs, cs = G.random_instance(rng, 24, [12], 50, [2])
        vs, cs = with_extras(vs, cs, rng, 10)
        arr, meta = run_gdba(vs, cs, {"increase_mode": "R"}, "min", 12, seed=8)
        G.save("gdba_rand_d12", arr, meta)


if __name__ == "__main__":
    main(sys.argv[1:])
