#!/usr/bin/env python
"""Generate tests/golden/dba_*.npz by running the UNMODIFIED reference DBA in lock-step.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_dba.py [fixture names]

Same method as tools/make_golden_gdba.py: the reference's own `DbaComputation` (pydcop/algorithms/dba.py:272) is
built through `build_computation(ComputationDef(node, algo))`, `message_sender` is replaced by a recorder and the
messages are delivered batch by batch.  One round is TWO batches: every ok message (phase 2k: each variable then
evaluates its values and posts its improve, dba.py:366-420), then every improve message (phase 2k + 1: each variable
then moves, raises its weights or stops, :504-562).  An End message is delivered with the batch it falls into.  The
reference has no stop_cycle: the driver stops delivering after n_cycles rounds.

Random draws (:343 start value, :412 pick among the best values) are injected from oracle/philox.py, keyed (seed;
variable, cycle) with cycle 0xffffffff at on_start and the computation's cycle_count after it.

Fixture keys: the constraint-hypergraph arrays of the GDBA fixtures (dom_size, factor_ptr, edge_var, table_off,
tables, var_ptr, var_con, init_value, var_rank) + per round k (row 0 = after on_start): value, cost (current_cost,
NaN while None), and the state each variable computed in the last phase it COMPLETED (a variable that finishes on an
End message completes nothing in that phase; what the improve messages that reached it before the End did to its
flags is not recorded):
  ok phase       eval (__cost__), improve, new_value (the value drawn, -1 without a draw), counter (as posted),
                 violated (per slot in var_con order: in _violated_constraints)
  both phases    can_move, qlm, consistent (as left by the later of the two)
  any time       weight (per slot), finish_phase (the phase of the first `finished()` call, 2^31 - 1 while live)
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
from pydcop.dcop.objects import Domain, Variable  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402
import pydcop.algorithms.dba as ref_dba  # noqa: E402

LIVE = 2 ** 31 - 1
INF = float("inf")


class _DbaRandom:
    """Replaces `random` in pydcop/algorithms/dba.py (stdlib; used :343, :412)."""

    @staticmethod
    def choice(seq):
        c = G._Ctx.comp
        cycle = philox.INIT_CYCLE if c._mode == "starting" else c.cycle_count
        seq = list(seq)
        _, w = philox.draw(G._Ctx.seed, G._Ctx.var, cycle)
        return seq[philox.choice_index(w, len(seq))]


def run_dba(variables, constraints, params, n_cycles, seed):
    variables, constraints = list(variables), list(constraints)
    arr, vidx = G.instance_arrays(variables, constraints)
    V, N = len(variables), n_cycles
    g = constraints_hypergraph.build_computation_graph(None, variables=variables, constraints=constraints)
    algo = AlgorithmDef.build_with_default_param("dba", dict(params), mode="min")
    comps, outbox = {}, []
    phase = [0]

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    doms = [list(v.domain) for v in variables]
    finish = np.full(V, LIVE, dtype=np.int32)
    nodes = {}
    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        # the first call: a stopping variable is put back in ok mode (dba.py:529) and an End message calls
        # finished() again
        c.finished = (lambda i=vidx[c.name]: finish.__setitem__(i, phase[0]) if finish[i] == LIVE else None)
        comps[c.name] = c
        nodes[c.name] = node
    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for v in variables:
        for c in comps[v.name].constraints:     # node.constraints order, dba.py:310
            var_con.append(cidx[c.name])
        var_ptr.append(len(var_con))
    arr["var_ptr"] = np.array(var_ptr, dtype=np.int32)
    arr["var_con"] = np.array(var_con, dtype=np.int32)
    arr["init_value"] = np.array([doms[i].index(v.initial_value) if v.initial_value is not None else -1
                                  for i, v in enumerate(variables)], dtype=np.int32)
    order = sorted(range(V), key=lambda i: variables[i].name)
    rank = np.zeros(V, dtype=np.int32)
    rank[order] = np.arange(V, dtype=np.int32)
    arr["var_rank"] = rank
    S = len(var_con)

    state = dict(eval=np.zeros(V, np.int64), improve=np.zeros(V, np.int64), new_value=np.full(V, -1, np.int32),
                 counter=np.zeros(V, np.int32), can_move=np.zeros(V, np.uint8), qlm=np.zeros(V, np.uint8),
                 consistent=np.zeros(V, np.uint8), violated=np.zeros(S, np.uint8))
    rows = {k: np.zeros((N + 1,) + a.shape, a.dtype) for k, a in state.items()}
    rows["value"] = np.zeros((N + 1, V), np.int32)
    rows["cost"] = np.full((N + 1, V), np.nan)
    rows["weight"] = np.zeros((N + 1, S), np.int32)
    rows["finish_phase"] = np.zeros((N + 1, V), np.int32)

    def flags(c, i):
        state["can_move"][i], state["qlm"][i] = c._can_move, c._quasi_local_minimum
        state["consistent"][i] = bool(c._consistent)

    orig_improve, orig_send_ok = ref_dba.DbaComputation.improve, ref_dba.DbaComputation._send_ok

    def improve_wrapper(self, relations):     # the ok phase completed
        out = orig_improve(self, relations)
        i = vidx[self.name]
        state["eval"][i], state["improve"][i] = self.__cost__, self._my_improve
        state["new_value"][i] = doms[i].index(self._new_value) if self._my_improve > 0 else -1
        state["counter"][i] = self._termination_counter
        s0 = var_ptr[i]
        state["violated"][s0:var_ptr[i + 1]] = 0
        for k in self._violated_constraints:
            state["violated"][s0 + k] = 1
        flags(self, i)
        return out

    def send_ok_wrapper(self):                # the improve phase completed
        out = orig_send_ok(self)
        flags(self, vidx[self.name])
        return out

    def snapshot(k):
        for i, v in enumerate(variables):
            c = comps[v.name]
            rows["value"][k, i] = doms[i].index(c.current_value)
            if c.current_cost is not None:
                rows["cost"][k, i] = c.current_cost
            rows["weight"][k, var_ptr[i]:var_ptr[i + 1]] = c.__constraints_weights__
        for key, a in state.items():
            rows[key][k] = a
        rows["finish_phase"][k] = finish

    def deliver(p):
        phase[0] = p
        batch, outbox[:] = list(outbox), []
        for s, d, m in batch:
            G._Ctx.var, G._Ctx.comp = vidx[d], comps[d]
            comps[d].on_message(s, m, 0)

    saved = ref_dba.random
    ref_dba.random = _DbaRandom
    ref_dba.DbaComputation.improve = improve_wrapper
    ref_dba.DbaComputation._send_ok = send_ok_wrapper
    G._Ctx.seed = seed
    try:
        t0 = time.perf_counter()
        for v in variables:
            G._Ctx.var, G._Ctx.comp = vidx[v.name], comps[v.name]
            comps[v.name].start()
        snapshot(0)
        for k in range(1, N + 1):
            deliver(2 * k)          # ok messages (and End messages) of round k
            deliver(2 * k + 1)      # improve messages (and End messages) of round k
            snapshot(k)
        dt = time.perf_counter() - t0
    finally:
        ref_dba.random = saved
        ref_dba.DbaComputation.improve = orig_improve
        ref_dba.DbaComputation._send_ok = orig_send_ok
    arr.update(rows)
    meta = dict(algo="dba", mode="min", params=dict(algo.params, stop_cycle=0), n_cycles=N, seed=seed,
                ref_seconds=dt, ref_var_updates_per_s=V * N / dt if dt > 0 else 0.0)
    return arr, meta


# ---- instances ---------------------------------------------------------------------------------------
def shuffled(rng, variables):
    """The variables in a random order, so that canonical order and name order differ (name ties decide)."""
    return [variables[i] for i in rng.permutation(len(variables))]


def with_extras(vs, cs, d=3):
    """A variable with a unary constraint only, and one without any constraint: neither has neighbours."""
    dom = Domain(f"dx{d}", "", list(range(d)))
    uno, iso = Variable("uno", dom), Variable("iso", dom)
    return vs + [uno, iso], cs + [NAryMatrixRelation([uno], np.array([INF] + [0.0] * (d - 1)), name="u_uno")]


def colouring(rng, n, d, n_edges, names=None, hard=INF):
    """A random graph colouring CSP: `hard` where the two colours are equal, 0 elsewhere."""
    dom = Domain(f"c{d}", "", list(range(d)))
    vs = [Variable(names[i] if names else f"x{i:02d}", dom) for i in range(n)]
    edges = set()
    while len(edges) < n_edges:
        a, b = sorted(int(x) for x in rng.choice(n, 2, replace=False))
        edges.add((a, b))
    t = np.where(np.eye(d, dtype=bool), hard, 0.0)
    cs = [NAryMatrixRelation([vs[a], vs[b]], t.copy(), name=f"e{a:02d}_{b:02d}") for a, b in sorted(edges)]
    return vs, cs


def ring(n, d, hard=INF):
    dom = Domain(f"c{d}", "", list(range(d)))
    vs = [Variable(f"r{i:02d}", dom) for i in range(n)]
    t = np.where(np.eye(d, dtype=bool), hard, 0.0)
    return vs, [NAryMatrixRelation([vs[i], vs[(i + 1) % n]], t.copy(), name=f"e{i:02d}") for i in range(n)]


def mixed(rng, n, levels):
    """Arities 1, 2 and 3 over domains 2, 3 and 4, entries drawn from `levels`."""
    doms = {d: Domain(f"m{d}", "", list(range(d))) for d in (2, 3, 4)}
    vs = [Variable(f"m{i:02d}", doms[(2, 3, 4)[i % 3]]) for i in range(n)]
    cs = []
    for j, a in enumerate([2, 3, 2, 1, 2, 3] * (n // 3)):
        sc = [vs[int(i)] for i in rng.choice(n, a, replace=False)]
        t = rng.choice(levels, size=tuple(len(v.domain) for v in sc))
        cs.append(NAryMatrixRelation(sc, t, name=f"k{j:02d}"))
    return vs, cs


def csp_yaml():
    """The reference's graph_coloring_csp.yaml, variables, constraints and scopes in name order (the loader's
    orders follow string hashing, which changes between processes)."""
    dcop = load_dcop_from_file([os.path.join(G.INSTANCES, "graph_coloring_csp.yaml")])
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


def k4():
    dom = Domain("c3", "", [0, 1, 2])
    vs = [Variable(f"k{i}", dom) for i in range(4)]
    t = np.where(np.eye(3, dtype=bool), INF, 0.0)
    return vs, [NAryMatrixRelation([vs[a], vs[b]], t.copy(), name=f"k{a}{b}") for a in range(4) for b in range(a + 1, 4)]


def named_colouring(seed, n, d, n_edges, **kw):
    rng = np.random.default_rng(seed)
    names = [f"n{int(x):02d}" for x in rng.permutation(n)]
    vs, cs = colouring(rng, n, d, n_edges, names=names, **kw)
    return with_extras(shuffled(rng, vs), cs, d)


def initial_values(seed):
    rng = np.random.default_rng(seed)
    vs, cs = colouring(rng, 14, 3, 18)
    vs2 = [Variable(v.name, v.domain, initial_value=list(v.domain)[i % 3]) for i, v in enumerate(vs)]
    by = {v.name: v for v in vs2}
    cs = [NAryMatrixRelation([by[v.name] for v in c.dimensions], c._m, name=c.name) for c in cs]
    return with_extras(vs2, cs)


def mixed_instance(seed, levels):
    rng = np.random.default_rng(seed)
    vs, cs = mixed(rng, 18, levels)
    return with_extras(shuffled(rng, vs), cs)


LEVELS_NEAR = np.array([0.0, 3.0, 9999.0, 9999.5, 10000.0, 10000.0, 20000.0, INF])
LEVELS_100 = np.array([0.0, 1.0, 99.0, 99.75, 100.0, 150.0, INF])

# name: (instance builder, params, rounds, seed, behaviours the fixture must show: test_dba_cpu.py)
CASES = {
    "dba_ref_gc_csp": (csp_yaml, {"infinity": 10000, "max_distance": 3}, 12, 2, ["all_finish"]),
    "dba_coloring_same_round": (lambda: named_colouring(3, 16, 3, 20), {"max_distance": 8}, 40, 5,
                                ["all_finish", "simultaneous_stop", "rank_decided"]),
    "dba_ring_flood": (lambda: with_extras(*ring(31, 2)), {"max_distance": 3}, 20, 6,
                       ["flood", "post_stop_move_d3", "eval_after_stop", "weights_grow"]),
    "dba_k4_unsat": (lambda: with_extras(*k4()), {"max_distance": 3}, 24, 6, ["no_stop", "weights_grow"]),
    "dba_mixed_near_infinity": (lambda: mixed_instance(7, LEVELS_NEAR), {"max_distance": 4}, 16, 8,
                                ["equal_infinity", "below_infinity", "inf_entries", "weights_grow"]),
    "dba_infinity_100": (lambda: mixed_instance(9, LEVELS_100), {"infinity": 100, "max_distance": 3}, 16, 10,
                         ["equal_infinity", "below_infinity", "weights_grow"]),
    "dba_max_distance_0": (lambda: named_colouring(11, 14, 3, 16), {"max_distance": 0}, 20, 12, ["no_stop"]),
    "dba_max_distance_1": (lambda: named_colouring(11, 14, 3, 16), {"max_distance": 1}, 20, 12, ["all_finish"]),
    "dba_initial_values": (lambda: initial_values(13), {"max_distance": 5}, 20, 14, ["initial_ignored"]),
    "dba_rand_d12": (lambda: named_colouring(15, 40, 12, 160, hard=10000.0), {"max_distance": 6}, 20, 16,
                     ["multi_draws"]),
}


def main(only=(), out_dir=None):
    only = set(only)
    if out_dir:
        G.GOLDEN = out_dir
    for name, (build, params, rounds, seed, _) in CASES.items():
        if only and name not in only:
            continue
        vs, cs = build()
        arr, meta = run_dba(vs, cs, params, rounds, seed)
        meta["shows"] = CASES[name][4]
        G.save(name, arr, meta)


if __name__ == "__main__":
    main(sys.argv[1:])
