#!/usr/bin/env python
"""Generate tests/golden/mgm2_*.npz by running the UNMODIFIED reference MGM-2 in lock-step.

TEST INFRASTRUCTURE (needs the reference source tree or its installed copy).  Run:
    python tools/make_golden_mgm2.py [fixture names]

Same method as oracle/make_golden_mgm.py: the reference's own `Mgm2Computation`
(pydcop/algorithms/mgm2.py:399) is built through `build_computation(ComputationDef(node, algo))`,
`message_sender` is replaced by a recorder and the messages are delivered batch by batch until
none is left.  A batch mixes cycles (a committed pair waits for its GO messages while its
neighbours already send the next values), so every record is keyed on the variable's own
`cycle_count`: the handlers of the gain phase and `_send_value` are wrapped.  A run without
`stop_cycle` is driven with stop_cycle = n_cycles + 1, which ends it after n_cycles rounds and
changes nothing before.

Random draws are injected from tests/_mgm2_oracle.py::draw (Philox, counter = (variable, cycle,
purpose, 0)); the lists the reference draws from are put in the canonical order first.

Fixture keys: the constraint-hypergraph arrays of the MGM fixtures (dom_size, factor_ptr,
edge_var, table_off, tables, var_ptr, var_con, unary, init_value, var_rank) + per round k
(row 0 = after on_start): value, cost (the reference's current_cost at the end of the round, NaN
while None), local_cost (the cost computed in the value phase), offerer, partner (position in the
variable's canonical neighbour list, or -1), committed, gain (potential_gain in the gain phase),
potential_value, go (a committed variable sent GO), cycle_count; finished at the end.
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
from _mgm2_oracle import (PURPOSE_FAVOR, PURPOSE_INIT, PURPOSE_OFFER, PURPOSE_PICK,  # noqa: E402
                          PURPOSE_VALUE, draw)

from pydcop.algorithms import AlgorithmDef, ComputationDef  # noqa: E402
from pydcop.computations_graph import constraints_hypergraph  # noqa: E402
from pydcop.dcop.objects import Domain, Variable, VariableWithCostDict  # noqa: E402
from pydcop.dcop.relations import NAryMatrixRelation  # noqa: E402
from pydcop.dcop.yamldcop import load_dcop_from_file  # noqa: E402
from pydcop.infrastructure.computations import build_computation  # noqa: E402
import pydcop.algorithms.mgm2 as ref_mgm2  # noqa: E402

M = ref_mgm2.Mgm2Computation


def canonical_neighbours(comp):
    seen = []
    for c in comp._constraints:
        for v in c.dimensions:
            if v.name != comp.variable.name and v.name not in seen:
                seen.append(v.name)
    return seen


class _Mgm2Random:
    """Replaces `random` in pydcop/algorithms/mgm2.py (stdlib; :469, :481, :755-757, :781, :821, :826)."""

    @staticmethod
    def _cycle(c):
        return philox.INIT_CYCLE if c._state is None else c.cycle_count

    @staticmethod
    def uniform(a, b):
        assert (a, b) == (0, 1)
        c = G._Ctx.comp
        purpose = {"value": PURPOSE_OFFER, "offer": PURPOSE_FAVOR}[c._state]
        return draw(G._Ctx.seed, G._Ctx.var, _Mgm2Random._cycle(c), purpose)[0]

    @staticmethod
    def choice(seq):
        c = G._Ctx.comp
        seq = list(seq)
        nbr = canonical_neighbours(c)
        if seq and hasattr(seq[0], "domain"):           # partner pick, mgm2.py:757
            seq = sorted(seq, key=lambda v: nbr.index(v.name))
            purpose = PURPOSE_OFFER
        elif seq and isinstance(seq[0], tuple):          # offer pick, mgm2.py:826
            own = list(c.variable.domain)

            def key(t):
                val_p, my_val, name = t
                return (nbr.index(name), list(c._neighbor_var(name).domain).index(val_p), own.index(my_val))
            seq = sorted(seq, key=key)
            purpose = PURPOSE_PICK
        else:                                            # values, in domain order
            purpose = PURPOSE_INIT if c._state is None else PURPOSE_VALUE
        _, w = draw(G._Ctx.seed, G._Ctx.var, _Mgm2Random._cycle(c), purpose)
        return seq[philox.choice_index(w, len(seq))]


def run_mgm2(variables, constraints, params, mode, n_cycles, seed):
    variables, constraints = list(variables), list(constraints)
    arr, vidx = G.instance_arrays(variables, constraints)
    V, N = len(variables), n_cycles
    g = constraints_hypergraph.build_computation_graph(None, variables=variables, constraints=constraints)
    run_params = dict(params)
    if not run_params.get("stop_cycle"):
        run_params["stop_cycle"] = N + 1
    algo = AlgorithmDef.build_with_default_param("mgm2", run_params, mode=mode)
    comps, outbox, finished = {}, [], set()

    def sender(s, d, m, prio=None, on_error=None):
        outbox.append((s, d, m))

    for node in g.nodes:
        c = build_computation(ComputationDef(node, algo))
        c.message_sender = sender
        c.finished = (lambda name=c.name: finished.add(name))
        comps[c.name] = c
    cidx = {c.name: i for i, c in enumerate(constraints)}
    var_ptr, var_con = [0], []
    for v in variables:
        for c in comps[v.name]._constraints:   # node.constraints order, mgm2.py:433
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

    rows = {k: np.full((N + 1, V), np.nan) for k in ("cost", "local_cost", "gain")}
    for k in ("value", "partner", "potential_value", "cycle_count"):
        rows[k] = np.full((N + 1, V), -1, dtype=np.int32)
    for k in ("offerer", "committed", "go"):
        rows[k] = np.zeros((N + 1, V), dtype=np.uint8)
    seen = np.zeros((N + 1, V), dtype=bool)

    def idx(c):
        return vidx[c.variable.name]

    orig_gain, orig_send = M._handle_gain_messages, M._send_value

    def gain_wrapper(self):
        i, k = idx(self), self.cycle_count
        nbr = canonical_neighbours(self)
        rows["local_cost"][k, i] = self.current_cost
        rows["offerer"][k, i] = self._is_offerer
        rows["partner"][k, i] = nbr.index(self._partner.name) if self._partner is not None else -1
        rows["committed"][k, i] = self._committed
        rows["gain"][k, i] = self._potential_gain
        rows["potential_value"][k, i] = doms[i].index(self._potential_value)
        # the GO message this round sends; _can_move is already cleared again when a GO
        # postponed from the partner is replayed inside the handler
        sent, post = [], self.post_msg

        def post_msg(target, msg, *a, **kw):
            if isinstance(msg, ref_mgm2.Mgm2GoMessage):
                sent.append(msg.go)
            return post(target, msg, *a, **kw)
        self.post_msg = post_msg
        try:
            orig_gain(self)
        finally:
            del self.post_msg
        rows["go"][k, i] = bool(sent and sent[0])

    def send_wrapper(self):
        i, k = idx(self), self.cycle_count
        rows["value"][k, i] = doms[i].index(self.current_value)
        if self.current_cost is not None:
            rows["cost"][k, i] = self.current_cost
        rows["cycle_count"][k, i] = k
        seen[k, i] = True
        orig_send(self)

    saved = ref_mgm2.random
    ref_mgm2.random = _Mgm2Random
    M._handle_gain_messages, M._send_value = gain_wrapper, send_wrapper
    G._Ctx.seed = seed
    try:
        t0 = time.perf_counter()
        for v in variables:
            G._Ctx.var, G._Ctx.comp = vidx[v.name], comps[v.name]
            comps[v.name].start()
        while outbox:
            batch, outbox[:] = list(outbox), []
            for s, d, m in batch:
                G._Ctx.var, G._Ctx.comp = vidx[d], comps[d]
                comps[d].on_message(s, m, 0)
        dt = time.perf_counter() - t0
    finally:
        ref_mgm2.random = saved
        M._handle_gain_messages, M._send_value = orig_gain, orig_send
    for i, v in enumerate(variables):
        c = comps[v.name]
        for k in range(N + 1):
            if seen[k, i]:
                continue
            if k == 0 or not c.neighbors_vars:   # no neighbours: the value of on_start, never sent
                rows["value"][k, i] = doms[i].index(c.current_value)
                rows["cost"][k, i] = c.current_cost
                rows["cycle_count"][k, i] = c.cycle_count
            else:                                # after the run stopped: the last state
                for key in ("value", "cost", "cycle_count"):
                    rows[key][k, i] = rows[key][k - 1, i]
    rows["cycle_count"][-1] = [comps[v.name].cycle_count for v in variables]
    arr.update(rows)
    arr["finished"] = np.array([v.name in finished for v in variables])
    meta = dict(algo="mgm2", mode=mode, params=dict(algo.params, stop_cycle=int(params.get("stop_cycle", 0))),
                n_cycles=N, seed=seed, ref_seconds=dt, ref_var_updates_per_s=V * N / dt if dt > 0 else 0.0)
    return arr, meta


def rebuild(constraints, variables):
    by_name = {v.name: v for v in variables}
    return [NAryMatrixRelation([by_name[v.name] for v in c.dimensions], c._m, name=c.name)
            for c in constraints]


def with_extras(vs, cs):
    """A variable whose only constraint is unary, and one without any constraint (own costs only)."""
    d3 = Domain("d3x", "", [0, 1, 2])
    uno = Variable("uno", d3)
    cs = cs + [NAryMatrixRelation([uno], np.array([2.0, 1.0, 1.0]), name="u_uno")]
    iso = VariableWithCostDict("iso", d3, {0: 0.5, 1: 0.25, 2: 0.25})
    return vs + [uno, iso], cs


CASES = {
    # name: (params, mode, arities, cost levels (0 = non-dyadic floats), var costs, initial values)
    "mgm2_default": ({}, "min", [2], 10, False, False),
    "mgm2_ties": ({}, "min", [2], 3, False, False),
    "mgm2_max": ({}, "max", [2], 4, False, False),
    "mgm2_mixed_arity": ({}, "min", [3, 2, 2, 1], 5, False, False),
    "mgm2_float": ({}, "min", [2, 2, 3], 0, False, False),
    # the favor rule only acts when the best offer's global gain EQUALS the unilateral gain: two cost
    # levels in max mode on instance seed 61 make that happen about once per cycle (the coin of
    # favor=no falls on both sides, coordinated commits), and every favor mode moves differently
    "mgm2_favor_unilateral": ({"favor": "unilateral"}, "max", [2], 2, False, False),
    "mgm2_favor_no": ({"favor": "no"}, "max", [2], 2, False, False),
    "mgm2_favor_coordinated": ({"favor": "coordinated"}, "max", [2], 2, False, False),
    "mgm2_threshold0": ({"threshold": 0.0}, "min", [2], 6, False, False),
    "mgm2_threshold1": ({"threshold": 1.0}, "min", [2], 6, False, False),
    "mgm2_initial_values": ({}, "min", [2], 6, False, True),
    "mgm2_var_costs": ({}, "min", [2, 2, 3], 6, True, False),
    "mgm2_stop8": ({"stop_cycle": 8}, "min", [2], 6, False, False),
    "mgm2_max_float": ({"favor": "coordinated"}, "max", [2, 3], 0, False, False),
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
        rng = np.random.default_rng(61 if name.startswith("mgm2_favor_") else 60)
        vs, cs = G.random_instance(rng, 26, [5, 4, 3], 40, arities)
        for c in cs:
            c._m[...] = (rng.integers(0, levels, size=c._m.shape) if levels
                         else np.round(rng.uniform(-3, 7, size=c._m.shape), 3))
        if init:
            vs2 = [Variable(v.name, v.domain, initial_value=(list(v.domain)[i % len(v.domain)] if i % 3 else None))
                   for i, v in enumerate(vs)]
            cs, vs = rebuild(cs, vs2), vs2
        if var_costs:
            vs2 = [VariableWithCostDict(v.name, v.domain, {x: float(rng.integers(0, 17)) / 8.0 for x in v.domain})
                   for v in vs]
            cs, vs = rebuild(cs, vs2), vs2
        vs, cs = with_extras(vs, cs)
        arr, meta = run_mgm2(vs, cs, params, mode, 12, seed=2468)
        G.save(name, arr, meta)
    if want("mgm2_gc10"):
        dcop = load_dcop_from_file([os.path.join(G.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
        arr, meta = run_mgm2(dcop.variables.values(), dcop.constraints.values(), {}, dcop.objective, 12, seed=91)
        G.save("mgm2_gc10", arr, meta)
    if want("mgm2_rand_d12"):
        rng = np.random.default_rng(61)
        vs, cs = G.random_instance(rng, 30, [12], 70, [2])
        arr, meta = run_mgm2(vs, cs, {}, "min", 10, seed=7)
        G.save("mgm2_rand_d12", arr, meta)


if __name__ == "__main__":
    main(sys.argv[1:])
