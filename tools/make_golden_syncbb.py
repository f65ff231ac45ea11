#!/usr/bin/env python
"""Generate tests/golden/syncbb_*.npz by running the UNMODIFIED reference SyncBB one message at a time.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_syncbb.py [fixture names]

The reference's own `SyncBBComputation` (pydcop/algorithms/syncbb.py:176) is built through
`build_computation(ComputationDef(node, algo))` over an `ordered_graph`, `message_sender` is replaced by a recorder,
and the messages are delivered from a FIFO queue.  SyncBB is a token walk: at most one message is ever in flight, so
this order is the only one the algorithm has.  Every computation is started in name order (only the first one posts).

Fixture keys: the instance arrays of the other fixtures (dom_size, factor_ptr, edge_var, table_off, tables, var_ptr,
var_con in node.constraints order, var_rank = position of the name in sorted order, unary = the variables' own costs,
canonical variable-major) + per delivered message k (row k, from 0):
  step_recv   canonical index of the receiver
  step_type   0 forward, 1 backward, 2 terminate
  step_plen   path length carried (0 for terminate)
  step_ub     bound carried (forward: the sender's, ignored by the receiver; terminate: NaN)
  ub          [k, V] every variable's upper_bound after the delivery
  sel         [k, V] every variable's last value_selection (domain index, -1 before any)
and final_sel (-1: no value), msg_count (every post, the start message included), n_steps, cycle_count (per
variable, the reference's new_cycle count) and finished (per variable, finished() was called).
Meta `error` holds the reference's exception where it raises (arity 3) and `dangling` the posts addressed to no
computation (one variable).
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden as G  # noqa: E402  (installs the reference shims)

from pydcop.algorithms import AlgorithmDef, ComputationDef  # noqa: E402
from pydcop.computations_graph import ordered_graph  # noqa: E402
from pydcop.dcop.objects import Domain, Variable, VariableWithCostDict  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation, constraint_from_str  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402

INF = float("inf")
TYPES = {"forward": 0, "backward": 1, "terminate": 2}


def run_syncbb(variables, constraints, mode, max_steps=200000):
    variables, constraints = list(variables), list(constraints)
    arr, vidx = G.instance_arrays(variables, constraints)
    V = len(variables)
    doms = [list(v.domain) for v in variables]
    unary = []
    for v in variables:
        unary += [float(v.cost_for_val(x)) if getattr(v, "has_cost", False) else 0.0 for x in v.domain]
    arr["unary"] = np.array(unary, dtype=np.float64)
    order = sorted(range(V), key=lambda i: variables[i].name)
    rank = np.zeros(V, dtype=np.int32)
    rank[order] = np.arange(V, dtype=np.int32)
    arr["var_rank"] = rank
    meta = dict(algo="syncbb", mode=mode, params={}, error=None, dangling=0)

    g = ordered_graph.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("syncbb", {}, mode=mode)
    comps, queue, posts = {}, [], [0]
    finished = np.zeros(V, dtype=np.uint8)

    def sender(s, d, m, prio=None, on_error=None):
        posts[0] += 1
        queue.append((s, d, m))

    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = (lambda i=vidx[c.name]: finished.__setitem__(i, 1))
        comps[c.name] = c
    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for v in variables:
        for c in comps[v.name].constraints:     # node.constraints order, syncbb.py:186
            var_con.append(cidx[c.name])
        var_ptr.append(len(var_con))
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_con"] = np.array(var_con, dtype=np.int32)

    def selection():
        out = np.full(V, -1, dtype=np.int32)
        for i, v in enumerate(variables):
            cv = comps[v.name].current_value
            if cv is not None:
                out[i] = doms[i].index(cv)
        return out

    recv, typ, plen, mub, ubs, sels = [], [], [], [], [], []
    t0 = time.perf_counter()
    try:
        for name in sorted(comps):
            comps[name].start()
        while queue and len(recv) < max_steps:
            s, d, m = queue.pop(0)
            if d is None:                       # syncbb.py:210 with one variable: no next computation
                meta["dangling"] += 1
                continue
            recv.append(vidx[d])
            typ.append(TYPES[m.type])
            plen.append(len(m.current_path) if m.type != "terminate" else 0)
            mub.append(float(m.ub) if m.type != "terminate" else np.nan)
            comps[d].on_message(s, m, 0)
            ubs.append([float(comps[v.name].upper_bound) for v in variables])
            sels.append(selection())
    except Exception as e:                      # noqa: BLE001  the reference's own error is the record
        while e.__context__ is not None:        # on_message re-raises a handler's error as KeyError(msg.type)
            e = e.__context__
        meta["error"] = f"{type(e).__name__}: {e}"
    dt = time.perf_counter() - t0
    if queue and meta["error"] is None and any(d is not None for _, d, _ in queue):
        raise RuntimeError(f"more than {max_steps} steps")
    n = len(ubs)                                # the delivery that raised is not a completed step
    recv, typ, plen, mub = recv[:n], typ[:n], plen[:n], mub[:n]
    arr.update(step_recv=np.array(recv, np.int32), step_type=np.array(typ, np.int8),
               step_plen=np.array(plen, np.int32), step_ub=np.array(mub, np.float64),
               ub=np.array(ubs, np.float64).reshape(n, V) if n else np.zeros((0, V)),
               sel=np.array(sels, np.int32).reshape(n, V) if n else np.zeros((0, V), np.int32),
               final_sel=selection(), msg_count=np.array(posts[0], np.int64), n_steps=np.array(n, np.int64),
               cycle_count=np.array([comps[v.name].cycle_count for v in variables], np.int64),
               finished=finished)
    meta.update(ref_seconds=dt, ref_steps_per_s=n / dt if dt > 0 else 0.0)
    return arr, meta


# ---- instances ---------------------------------------------------------------------------------------
def toy():
    """The reference's unit-test problem (tests/unit/test_algorithms_syncbb.py:build_pb)."""
    v_a, v_b, v_c, v_d = (Variable(n, ["R", "G"]) for n in ("vA", "vB", "vC", "vD"))
    c1 = constraint_from_str("c1", "{('R', 'G'): 8, ('R', 'R'): 5, ('G', 'G'): 3, ('G', 'R'): 20}[(vA, vB)]",
                             [v_a, v_b])
    c2 = constraint_from_str("c2", "{('R', 'G'): 10, ('R', 'R'): 5, ('G', 'G'): 3, ('G', 'R'): 20}[(vA, vC)]",
                             [v_a, v_c])
    c3 = constraint_from_str("c3", "{('R', 'G'): 4, ('R', 'R'): 5, ('G', 'G'): 3, ('G', 'R'): 3}[(vB, vC)]",
                             [v_b, v_c])
    c4 = constraint_from_str("c4", "{('R', 'G'): 8, ('R', 'R'): 3, ('G', 'G'): 3, ('G', 'R'): 10}[(vB, vD)]",
                             [v_b, v_d])
    return [v_a, v_b, v_c, v_d], [c1, c2, c3, c4]


def from_yaml(fname):
    """A reference instance, variables, constraints and scopes in name order (the loader's orders follow string
    hashing, which changes between processes)."""
    dcop = load_dcop_from_file([os.path.join(G.INSTANCES, fname)])
    vs = [dcop.variables[n] for n in sorted(dcop.variables)]
    cs = []
    for n in sorted(dcop.constraints):
        c = dcop.constraints[n]
        dims = sorted(c.dimensions, key=lambda v: v.name)
        t = np.zeros(tuple(len(v.domain) for v in dims))
        for idx in np.ndindex(*t.shape):
            t[idx] = c(**{v.name: list(v.domain)[i] for v, i in zip(dims, idx)})
        cs.append(NAryMatrixRelation(dims, t, name=n))
    return vs, cs


def random_binary(seed, n, d, n_edges, levels, names=None, shuffle=False, dom_sizes=None):
    """Random binary constraints with entries drawn from `levels`; `names` gives the variables other names than
    their canonical order, `shuffle` lists them in a random order."""
    rng = np.random.default_rng(seed)
    sizes = dom_sizes if dom_sizes is not None else [d] * n
    vs = [Variable(names[i] if names else f"x{i:02d}", Domain(f"d{sizes[i]}", "", list(range(sizes[i]))))
          for i in range(n)]
    edges = set()
    while len(edges) < n_edges:
        a, b = (int(x) for x in rng.choice(n, 2, replace=False))
        edges.add((a, b))
    cs = [NAryMatrixRelation([vs[a], vs[b]], rng.choice(levels, size=(len(vs[a].domain), len(vs[b].domain))),
                             name=f"c{j:02d}") for j, (a, b) in enumerate(sorted(edges))]
    if shuffle:
        vs = [vs[i] for i in rng.permutation(n)]
    return vs, cs


def with_ignored(seed):
    """Unary constraints on every variable and variable costs on half of them: SyncBB reads neither."""
    vs, cs = random_binary(seed, 7, 3, 9, np.arange(10.0))
    rng = np.random.default_rng(seed + 1)
    vs2 = [VariableWithCostDict(v.name, v.domain, {x: float(rng.integers(0, 20)) for x in v.domain})
           if i % 2 == 0 else v for i, v in enumerate(vs)]
    by = {v.name: v for v in vs2}
    cs2 = [NAryMatrixRelation([by[v.name] for v in c.dimensions], c._m, name=c.name) for c in cs]
    cs2 += [NAryMatrixRelation([v], rng.integers(0, 30, size=len(v.domain)).astype(float), name=f"u_{v.name}")
            for v in vs2]
    return vs2, cs2


def with_isolated(seed):
    vs, cs = random_binary(seed, 6, 3, 7, np.arange(6.0))
    return vs + [Variable("x03b", Domain("d3", "", [0, 1, 2]))], cs


def infeasible():
    """Two variables that must differ and equal at once: every full assignment costs inf."""
    dom = Domain("c2", "", [0, 1])
    a, b, c = Variable("a", dom), Variable("b", dom), Variable("c", dom)
    eq = np.where(np.eye(2, dtype=bool), 0.0, INF)
    ne = np.where(np.eye(2, dtype=bool), INF, 0.0)
    return [a, b, c], [NAryMatrixRelation([a, b], eq, name="ab_eq"), NAryMatrixRelation([a, b], ne, name="ab_ne"),
                       NAryMatrixRelation([b, c], ne, name="bc_ne")]


def arity3():
    dom = Domain("c2", "", [0, 1])
    a, b, c = Variable("a", dom), Variable("b", dom), Variable("c", dom)
    return [a, b, c], [NAryMatrixRelation([a, b], np.arange(4.0).reshape(2, 2), name="ab"),
                       NAryMatrixRelation([a, b, c], np.arange(8.0).reshape(2, 2, 2), name="abc")]


def one_var():
    a = Variable("a", Domain("c3", "", [0, 1, 2]))
    return [a], [NAryMatrixRelation([a], np.array([3.0, 1.0, 2.0]), name="u_a")]


def partial_accept():
    """The first random instance (seed 100 on) whose SyncBB answer is not the optimum: a candidate that fails at a
    later path element is accepted with its partial cost, and the bound then prunes the optimum."""
    import itertools
    for seed in range(100, 400):
        vs, cs = random_binary(seed, 5, 3, 6, np.arange(8.0))
        arr, meta = run_syncbb(vs, cs, "min")
        best = min(sum(float(c(**{v.name: asg[vs.index(v)] for v in c.dimensions})) for c in cs)
                   for asg in itertools.product(*[list(v.domain) for v in vs]))
        got = {v.name: list(v.domain)[int(arr["final_sel"][i])] for i, v in enumerate(vs)}
        cost = sum(float(c(**{v.name: got[v.name] for v in c.dimensions})) for c in cs)
        if cost != best:
            meta.update(seed=seed, optimum=best, found=cost)
            return arr, meta
    raise RuntimeError("no instance found")


NAMES = [f"n{i:02d}" for i in (7, 2, 9, 0, 5, 3, 8, 1, 6, 4)]
FLOATS = np.array([0.1, 0.3, 0.7, 1.1, 1.7, 2.9, 0.2, 3.3])
WITH_INF = np.array([0.0, 1.0, 2.0, 4.0, 7.0, INF, INF])

# name: (instance builder, mode, behaviours the fixture must show: test_syncbb_cpu.py)
CASES = {
    "syncbb_toy_min": (toy, "min", ["toy_min"]),
    "syncbb_toy_max": (toy, "max", ["toy_max", "exhaustive"]),
    "syncbb_tuto": (lambda: from_yaml("graph_coloring_tuto.yaml"), "min", ["tuto"]),
    "syncbb_gc_csp": (lambda: from_yaml("graph_coloring_csp.yaml"), "min", ["inf_entries"]),
    "syncbb_partial_accept": (None, "min", ["partial_accept"]),
    "syncbb_floats": (lambda: random_binary(11, 8, 3, 12, FLOATS), "min", ["non_dyadic"]),
    "syncbb_floats_max": (lambda: random_binary(12, 6, 3, 8, FLOATS), "max", ["exhaustive", "non_dyadic"]),
    "syncbb_inf": (lambda: random_binary(13, 8, 3, 12, WITH_INF), "min", ["inf_entries", "inf_prunes"]),
    "syncbb_ignored": (lambda: with_ignored(14), "min", ["ignored"]),
    "syncbb_name_order": (lambda: random_binary(15, 10, 3, 14, np.arange(12.0), names=NAMES, shuffle=True), "min",
                          ["name_order"]),
    "syncbb_mixed_domains": (lambda: random_binary(16, 8, 0, 12, np.arange(9.0), dom_sizes=[2, 4, 3, 5, 2, 3, 4, 2]),
                             "min", []),
    "syncbb_isolated": (lambda: with_isolated(17), "min", ["isolated"]),
    "syncbb_infeasible": (infeasible, "min", ["infeasible"]),
    "syncbb_arity3": (arity3, "min", ["error"]),
    "syncbb_one_var": (one_var, "min", ["dangling"]),
}


def main(only=(), out_dir=None):
    only = set(only)
    if out_dir:
        G.GOLDEN = out_dir
    for name, (build, mode, shows) in CASES.items():
        if only and name not in only:
            continue
        if build is None:
            arr, meta = partial_accept()
        else:
            vs, cs = build()
            arr, meta = run_syncbb(vs, cs, mode)
        meta["shows"] = shows
        meta["var_names"] = [str(x) for x in arr["var_names"]]
        G.save(name, arr, meta)


if __name__ == "__main__":
    main(sys.argv[1:])
