#!/usr/bin/env python
"""Generate tests/golden/dpop_*.npz by running the UNMODIFIED reference DPOP.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_dpop.py [fixture names]

The reference's own `DpopAlgo` (pydcop/algorithms/dpop.py:115) is built through
`build_computation(ComputationDef(node, algo))` on the nodes of its own
`pseudotree.build_computation_graph`.  `message_sender` is replaced by a recorder.  Every computation
is started (leaves send their UTIL, isolated variables choose), then UTILs are delivered to each parent
in the pseudo-tree's children order, nodes taken children first, and finally the VALUE messages in the
order they are sent.

NumPy 2 removed `ndarray.itemset`, which `NAryMatrixRelation.set_value_for_assignment` uses with a dict
assignment (relations.py:857); the tool restates that branch with an item assignment, which converts the
value to the matrix's dtype exactly as `itemset` did.

Fixture keys: the instance arrays (dom_size, factor_ptr, edge_var, table_off, tables, unary, var_names),
the reference's tree (parent, children / pseudo_parents / pseudo_children as ptr + idx CSR, owner per
constraint), every UTIL message (util_var_ptr / util_var: sender's dimension variables in the message's
order, util_ptr / util: its entries row-major over them; a root's rows are empty), every VALUE message
received (value_ptr / value_var / value_val: per receiver, in message order) and the final value index and
cost of every variable.  meta["error"] names the exception when the reference raises (the infeasible
fixture records that, not a trajectory).
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden as G  # noqa: E402  (installs the reference shims)

from pydcop.algorithms import AlgorithmDef, ComputationDef  # noqa: E402
from pydcop.computations_graph import pseudotree  # noqa: E402
from pydcop.dcop.objects import Domain, Variable, VariableWithCostDict  # noqa: E402
from pydcop.dcop import relations  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402

_orig_set = NAryMatrixRelation.set_value_for_assignment


def _set_value_for_assignment(self, var_values, rel_value):
    if isinstance(var_values, dict):
        values = [var_values[v.name] for v in self._variables]
        _, s = self._slice_matrix([v.name for v in self._variables], values)
        matrix = np.copy(self._m)
        matrix[s] = rel_value
        return NAryMatrixRelation(self._variables, matrix, name=self.name)
    return _orig_set(self, var_values, rel_value)


NAryMatrixRelation.set_value_for_assignment = _set_value_for_assignment
assert relations.NAryMatrixRelation is NAryMatrixRelation


def csr(lists):
    ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    idx = np.array([y for x in lists for y in x], dtype=np.int32)
    return ptr, idx


def run_dpop(variables, constraints, mode):
    variables, constraints = list(variables), list(constraints)
    arr, vidx = G.instance_arrays(variables, constraints)
    arr["unary"] = np.array([float(v.cost_for_val(x)) if hasattr(v, "cost_for_val") else 0.0
                             for v in variables for x in v.domain])
    V = len(variables)
    doms = [list(v.domain) for v in variables]
    g = pseudotree.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("dpop", {}, mode=mode)
    comps, outbox, utils, values = {}, [], {}, {i: [] for i in range(V)}

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))
        if m.type == "UTIL":
            utils[vidx[s]] = ([vidx[v.name] for v in m.content.dimensions], np.asarray(m.content._m, dtype=np.float64))
        else:
            values[vidx[d]].append([(vidx[v.name], doms[vidx[v.name]].index(x)) for v, x in zip(*m.content)])

    rel = {}
    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = lambda: None
        comps[c.name] = c
        rel[vidx[c.name]] = pseudotree.get_dfs_relations(node)
    name = [v.name for v in variables]
    parent = np.array([vidx[rel[i][0]] if rel[i][0] is not None else -1 for i in range(V)], dtype=np.int32)
    children = [[vidx[x] for x in rel[i][2]] for i in range(V)]
    cidx = {c.name: f for f, c in enumerate(constraints)}
    owner = np.full(len(constraints), -1, dtype=np.int32)
    for i in range(V):
        for c in comps[name[i]]._constraints:
            owner[cidx[c.name]] = i
    arr["parent"] = parent
    arr["children_ptr"], arr["children_idx"] = csr(children)
    arr["pseudo_parents_ptr"], arr["pseudo_parents_idx"] = csr([[vidx[x] for x in rel[i][1]] for i in range(V)])
    arr["pseudo_children_ptr"], arr["pseudo_children_idx"] = csr([[vidx[x] for x in rel[i][3]] for i in range(V)])
    arr["owner"] = owner
    roots = [r.variable.name for r in g.roots]
    order = []                                   # preorder of the reference's trees
    for r in roots:
        stack = [vidx[r]]
        while stack:
            u = stack.pop()
            order.append(u)
            stack.extend(reversed(children[u]))
    error = None
    t0 = time.perf_counter()
    try:
        for v in variables:
            comps[v.name].start()
        pending = {}

        def drain():
            for s, d, m in outbox:
                pending[(s, d, m.type)] = m
            outbox[:] = []
        drain()
        for u in reversed(order):
            for c in children[u]:
                comps[name[u]].on_message(name[c], pending.pop((name[c], name[u], "UTIL")), 0)
                drain()
        queue = [k for k in pending]
        while queue:
            s, d, typ = queue.pop(0)
            comps[d].on_message(s, pending.pop((s, d, typ)), 0)
            before = set(pending)
            drain()
            queue += [k for k in pending if k not in before]
    except Exception as e:  # noqa: BLE001 — the unresolved case: the reference's IndexError is the fixture
        error = type(e).__name__
    dt = time.perf_counter() - t0
    uv = [utils.get(i, ([], np.zeros(0)))[0] for i in range(V)]
    arr["util_var_ptr"], arr["util_var"] = csr(uv)
    ut = [utils.get(i, ([], np.zeros(0)))[1].reshape(-1) if i in utils else np.zeros(0) for i in range(V)]
    arr["util_ptr"] = np.concatenate([[0], np.cumsum([len(x) for x in ut])]).astype(np.int64)
    arr["util"] = np.concatenate(ut) if ut else np.zeros(0)
    msgs = [m for i in range(V) for m in values[i]]
    arr["value_ptr"] = np.concatenate([[0], np.cumsum([len(values[i]) for i in range(V)])]).astype(np.int32)
    arr["value_msg_ptr"], flat = csr([[k for k, _ in m] for m in msgs])
    arr["value_var"] = flat
    arr["value_val"] = np.array([x for m in msgs for _, x in m], dtype=np.int32)
    if error is None:
        arr["value"] = np.array([doms[i].index(comps[name[i]].current_value) for i in range(V)], dtype=np.int32)
        arr["cost"] = np.array([float(comps[name[i]].current_cost) for i in range(V)])
    meta = dict(algo="dpop", mode=mode, error=error, ref_seconds=dt, roots=[vidx[r] for r in roots])
    return arr, meta


def table(rng, shape, kind):
    if kind == "float":
        return np.round(rng.uniform(-5, 5, size=shape), 4) + 1 / 3
    if kind == "ties":
        return rng.integers(0, 2, size=shape).astype(float)
    if kind == "hard":
        m = rng.integers(0, 4, size=shape).astype(float)
        m[rng.uniform(size=shape) < 0.45] = np.inf
        return m
    if kind == "big":
        m = rng.integers(0, 6, size=shape).astype(float)
        hit = rng.uniform(size=shape) < 0.5
        m[hit] = 3.0e9 + rng.integers(0, 1000, size=shape)[hit]
        return m
    return rng.integers(0, 10, size=shape).astype(float)


def random_case(rng, n_vars, doms, scopes, kind, var_costs=False):
    ds = {}
    vs = []
    for i in range(n_vars):
        d = int(doms[i % len(doms)])
        ds.setdefault(d, Domain(f"d{d}", "", list(range(d))))
        if var_costs:
            vs.append(VariableWithCostDict(f"v{i:02d}", ds[d], {x: float(rng.integers(0, 5)) / 3 for x in range(d)}))
        else:
            vs.append(Variable(f"v{i:02d}", ds[d]))
    cs = [NAryMatrixRelation([vs[i] for i in s], table(rng, tuple(len(vs[i].domain) for i in s), kind),
                             name=f"c{j:02d}") for j, s in enumerate(scopes)]
    return vs, cs


def random_scopes(rng, n_vars, n_cons, arities):
    out = []
    for j in range(n_cons):
        a = int(arities[j % len(arities)])
        out.append([int(x) for x in rng.choice(n_vars, size=a, replace=False)])
    return out


def star_scopes(rng, n_vars, extra):
    """A hub with several subtrees (nodes with >= 3 children) plus a few random back-edges."""
    out = [[0, i] for i in range(1, 5)]
    for i in range(5, n_vars):
        out.append([int(rng.integers(1, i)), i])
    return out + random_scopes(rng, n_vars, extra, [2])


def components_case(rng):
    d3 = Domain("d3", "", [0, 1, 2])
    vs = [Variable(f"a{i}", d3) for i in range(6)] + [Variable(f"b{i}", d3) for i in range(5)]
    vs.append(VariableWithCostDict("iso", d3, {0: 0.5, 1: 0.25, 2: 0.25}))
    vs.append(Variable("plain", d3))
    uno = Variable("uno", d3)
    vs.append(uno)
    cs = []
    for k, (lo, n) in enumerate(((0, 6), (6, 5))):
        for i in range(1, n):
            p = lo + int(rng.integers(0, i))
            cs.append(NAryMatrixRelation([vs[p], vs[lo + i]], table(rng, (3, 3), "int"), name=f"k{k}_{i}"))
    cs.append(NAryMatrixRelation([vs[0], vs[2], vs[4]], table(rng, (3, 3, 3), "int"), name="k0_t"))
    cs.append(NAryMatrixRelation([uno], np.array([2.0, 1.0, 1.5]), name="u_uno"))
    cs.append(NAryMatrixRelation([vs[1]], np.array([0.5, 0.0, 0.25]), name="u_a1"))
    return vs, cs


def ref_file(name):
    dcop = load_dcop_from_file([os.path.join(G.INSTANCES, name)])
    return list(dcop.variables.values()), list(dcop.constraints.values()), dcop.objective


def cases():
    out = {}
    for n in ("graph_coloring_10_4_15_0.1.yml", "graph_coloring_tuto_max.yaml", "graph_coloring_csp.yaml",
              "graph_coloring_seperate_costs.yaml", "graph_coloring_10_4_15_0.1_capa_costs.yml",
              "graph_coloring_tuto.yaml"):
        key = "dpop_ref_" + n.split(".yaml")[0].split(".yml")[0].replace("graph_coloring", "gc").replace(".", "_")
        out[key] = lambda n=n: ref_file(n)

    def rnd(seed, n, doms, scopes_fn, kind, mode="min", var_costs=False):
        def f():
            rng = np.random.default_rng(seed)
            vs, cs = random_case(rng, n, doms, scopes_fn(rng), kind, var_costs)
            return vs, cs, mode
        return f
    out["dpop_float_star"] = rnd(1, 16, [3, 4], lambda r: star_scopes(r, 16, 6), "float", var_costs=True)
    out["dpop_float_max"] = rnd(2, 14, [3], lambda r: star_scopes(r, 14, 5), "float", mode="max")
    out["dpop_nary"] = rnd(3, 10, [2, 3, 4], lambda r: random_scopes(r, 10, 9, [3, 4, 2]), "int")
    out["dpop_ties"] = rnd(4, 14, [3], lambda r: star_scopes(r, 14, 6), "ties")
    out["dpop_hard"] = rnd(5, 12, [3], lambda r: star_scopes(r, 12, 4), "hard")
    out["dpop_big_costs"] = rnd(6, 12, [3], lambda r: star_scopes(r, 12, 4), "big")
    out["dpop_components"] = lambda: (*components_case(np.random.default_rng(7)), "min")

    def infeasible():
        d2 = Domain("d2", "", [0, 1])
        a, b, c = Variable("a", d2), Variable("b", d2), Variable("c", d2)
        inf = np.inf
        return [a, b, c], [NAryMatrixRelation([a, b], np.array([[inf, inf], [inf, inf]]), name="ab"),
                           NAryMatrixRelation([b, c], np.array([[0.0, 1.0], [2.0, 3.0]]), name="bc")], "min"
    out["dpop_infeasible"] = infeasible
    return out


def main(only=()):
    only = set(only)
    for name, make in cases().items():
        if only and name not in only:
            continue
        vs, cs, mode = make()
        arr, meta = run_dpop(vs, cs, mode)
        G.save(name, arr, meta)
        print(f"  error={meta['error']} roots={len(meta['roots'])}")


if __name__ == "__main__":
    main(sys.argv[1:])
