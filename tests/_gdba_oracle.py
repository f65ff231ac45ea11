"""GDBA restated in plain Python: the oracle of the `gdba_*` fixtures and of the GDBA kernels.
TEST INFRASTRUCTURE ONLY (the product package never imports it).

One `step()` is one GDBA round of pydcop/algorithms/gdba.py for every variable at once (ok phase
:352-387, improve phase :493-541), in the precision of `dtype` (np.float32 scalars round every
operation to f32).

Evaluation (compute_eval_value, :428-461): the constraints in `node.constraints` order; after the
effective cost of constraint k the variable costs of every distinct variable seen in the scopes of
constraints 0..k are added again (own variable at its CURRENT value).  That prefix term is summed
here as own cost, then the neighbours in order of first appearance; the reference sums a set in an
undefined order, so fixtures use integer or dyadic variable costs.
  eval(x) = ((((0 + eff_0(x)) + vc_0) + eff_1(x)) + vc_1) + ...
  eff_k(x) = base + m (modifier "A", m from 0) | base * m (modifier "M", m from 1)

Modifiers (_increase_cost, :627-654): the reference keys its writes on the variable's whole
neighbourhood, its reads on the constraint's scope, so E / R / C writes are only ever read on a
constraint whose scope is exactly {variable} + all its neighbours ("spanning"); elsewhere they
change nothing.  T increments every entry of the constraint: one count per (variable, constraint).
State here: `cnt[v][k]` (T) and `tab[v][k]` (an int table over the constraint's entries for a
spanning slot under E / R / C, None otherwise).

Random draws are injected as MGM's: Philox4x32-10 with counter (canonical variable id, cycle, 0, 0)
(oracle/philox.py `draw`), cycle = 0xffffffff for the start value, else the 1-based round; best
values are drawn from in domain order.
"""
import numpy as np

import philox
from _mgm2_oracle import neighbour_lists, var_constraints

MODIFIERS = ("A", "M")
VIOLATIONS = ("NZ", "NM", "MX")
INCREASE_MODES = ("E", "R", "C", "T")


class GdbaOracle:
    """Lock-step GDBA.  State after `init()` == fixture row 0, after n `step()` == row n."""

    def __init__(self, inst, dtype=np.float64, mode="min", modifier="A", violation="NZ", increase_mode="E",
                 stop_cycle=0, seed=0, var_id=None, **_ignored):
        if modifier not in MODIFIERS or violation not in VIOLATIONS or increase_mode not in INCREASE_MODES:
            raise ValueError(f"invalid parameters {modifier!r} {violation!r} {increase_mode!r}")
        self.T = np.float64 if np.dtype(dtype) == np.float64 else np.float32
        self.mode_max = mode == "max"
        self.modifier, self.violation, self.increase_mode = modifier, violation, increase_mode
        self.base_mod = 0 if modifier == "A" else 1
        self.stop_cycle, self.seed = int(stop_cycle or 0), int(seed)
        self.dom = [int(x) for x in inst["dom_size"]]
        V = self.V = len(self.dom)
        fp = [int(x) for x in inst["factor_ptr"]]
        ev = [int(x) for x in inst["edge_var"]]
        tsize = [int(np.prod([self.dom[u] for u in ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)]
        self.toff = [0] + list(np.cumsum(tsize, dtype=np.int64))
        if "table_off" in inst and inst["table_off"] is not None:
            self.toff = [int(x) for x in inst["table_off"]]
        self.tsize = tsize
        self.tables = np.ascontiguousarray(inst["tables"], dtype=self.T)
        self.scope = [ev[fp[f]:fp[f + 1]] for f in range(len(fp) - 1)]
        self.strides = []
        for sc in self.scope:
            st, acc = [0] * len(sc), 1
            for i in range(len(sc) - 1, -1, -1):
                st[i] = acc
                acc *= self.dom[sc[i]]
            self.strides.append(st)
        var_ptr = [int(x) for x in inst["var_ptr"]]
        var_con = [int(x) for x in var_constraints(inst)]
        self.cons = [var_con[var_ptr[v]:var_ptr[v + 1]] for v in range(V)]
        self.nbrs = neighbour_lists(self.dom, fp, ev, var_ptr, var_con)
        uoff = np.concatenate([[0], np.cumsum(self.dom)]).astype(np.int64)
        unary = np.asarray(inst["unary"], dtype=self.T) if "unary" in inst else np.zeros(int(uoff[-1]), self.T)
        self.unary = [unary[uoff[v]:uoff[v + 1]] for v in range(V)]
        iv = inst["init_value"] if "init_value" in inst else None
        self.init_value = [int(x) for x in iv] if iv is not None else [-1] * V
        rank = inst["var_rank"] if "var_rank" in inst else None
        self.rank = [int(x) for x in rank] if rank is not None else list(range(V))
        self.var_id = [int(x) for x in var_id] if var_id is not None else list(range(V))
        # violation reference value per constraint (min / max of the BASE table, :252-274)
        self.tmin = [self.tables[self.toff[f]:self.toff[f] + tsize[f]].min() for f in range(len(tsize))]
        self.tmax = [self.tables[self.toff[f]:self.toff[f] + tsize[f]].max() for f in range(len(tsize))]
        self.span = [[bool(self.nbrs[v]) and set(self.scope[f]) == {v, *self.nbrs[v]} for f in self.cons[v]]
                     for v in range(V)]
        self.cycle = 0

    # -- pieces of the reference computation --------------------------------------------------
    def _index(self, f, val):
        i = 0
        for u, s in zip(self.scope[f], self.strides[f]):
            i += val[u] * s
        return i

    def modifier_at(self, v, k, i):
        """Modifier of slot k of v at entry i of its constraint, as _get_modifier_for_assignment reads it."""
        m = self.base_mod + self.cnt[v][k]
        if self.tab[v][k] is not None:
            m += int(self.tab[v][k][i])
        return m

    def eff_cost(self, v, k, val):
        """_eff_cost (:574-597) of slot k of v at the assignment `val`."""
        f = self.cons[v][k]
        i = self._index(f, val)
        c = self.tables[self.toff[f] + i]
        m = self.T(self.modifier_at(v, k, i))
        return c + m if self.modifier == "A" else c * m

    def is_violated(self, v, k, val):
        """_is_violated (:552-572), on the base table."""
        f = self.cons[v][k]
        c = self.tables[self.toff[f] + self._index(f, val)]
        if self.violation == "NZ":
            return bool(c != 0)
        if self.violation == "NM":
            return bool(c != self.tmin[f])
        return bool(c == self.tmax[f])

    def var_cost_terms(self, v, val):
        """The prefix variable-cost term added after each constraint (own variable at val[v])."""
        out, seen = [], {v}
        acc = self.unary[v][val[v]]
        for f in self.cons[v]:
            for u in self.scope[f]:
                if u not in seen:
                    seen.add(u)
                    acc = acc + self.unary[u][val[u]]
            out.append(acc)
        return out

    def eval_value(self, v, x, val, vc=None):
        """compute_eval_value(x) (:428-461) with the other variables at `val`."""
        vc = self.var_cost_terms(v, val) if vc is None else vc
        work = list(val)
        work[v] = x
        acc = self.T(0)
        for k in range(len(self.cons[v])):
            acc = (acc + self.eff_cost(v, k, work)) + vc[k]
        return acc

    def best_values(self, v, val):
        """_compute_best_improvement (:395-417): (best values in domain order, best evaluation)."""
        vc = self.var_cost_terms(v, val)
        best, vals = None, []
        for x in range(self.dom[v]):
            c = self.eval_value(v, x, val, vc)
            if best is None or (c > best if self.mode_max else c < best):
                best, vals = c, [x]
            elif c == best:
                vals.append(x)
        return vals, best

    def increase_cost(self, v, k, val):
        """_increase_cost (:627-654) of slot k of v, the neighbours at `val`."""
        if self.increase_mode == "T":
            self.cnt[v][k] += 1
            return
        tab = self.tab[v][k]
        if tab is None:          # the write's key names the whole neighbourhood: never read here
            return
        f = self.cons[v][k]
        j = self.scope[f].index(v)
        sv, d = self.strides[f][j], self.dom[v]
        i = self._index(f, val)
        if self.increase_mode == "E":
            tab[i] += 1
        elif self.increase_mode == "R":
            i0 = i - val[v] * sv
            for x in range(d):
                tab[i0 + x * sv] += 1
        else:                    # C: every entry with the own value at val[v]
            idx = np.arange(self.tsize[f])
            tab[(idx // sv) % d == val[v]] += 1

    # -- lifecycle -----------------------------------------------------------------------------
    def init(self):
        V = self.V
        self.val = [0] * V
        self.cost = [None] * V
        for v in range(V):
            if self.nbrs[v]:
                if self.init_value[v] >= 0:
                    self.val[v] = self.init_value[v]
                else:
                    _, w = philox.draw(self.seed, self.var_id[v], philox.INIT_CYCLE)
                    self.val[v] = philox.choice_index(w, self.dom[v])
            else:  # optimal_cost_value over the variable's own costs, then finished (:304-315)
                c = self.unary[v]
                x = int(len(c) - 1 - np.argmax(c[::-1])) if self.mode_max else int(np.argmin(c))
                self.val[v], self.cost[v] = x, c[x]
        self.cnt = [[0] * len(self.cons[v]) for v in range(V)]
        self.tab = [[np.zeros(self.tsize[f], dtype=np.int64) if (self.span[v][k] and self.increase_mode != "T")
                     else None for k, f in enumerate(self.cons[v])] for v in range(V)]
        self.cycle = 0
        self.last = None
        self.stats = dict(breakouts=0, span_increases=0, other_breakout_slots=0, rank_decided=0,
                          multi_draws=0, max_breakouts_next_to_improving=0)
        return self

    @property
    def finished(self):
        """stop_cycle with mgm_gpu's convention: a run ends when rounds done + 1 >= stop_cycle."""
        return bool(self.stop_cycle and self.cycle + 1 >= self.stop_cycle)

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self._round(self.cycle + 1)
            self.cycle += 1
        return self

    def _improving(self, g):
        return g < 0 if self.mode_max else g > 0

    def _round(self, cyc):
        V, val = self.V, self.val
        conn = [v for v in range(V) if self.nbrs[v]]
        cost, improve, new_value = list(self.cost), [None] * V, list(val)
        violated = [[False] * len(self.cons[v]) for v in range(V)]
        # ok phase (:352-387)
        for v in conn:
            violated[v] = [self.is_violated(v, k, val) for k in range(len(self.cons[v]))]
            vc = self.var_cost_terms(v, val)
            cst = self.eval_value(v, val[v], val, vc)
            vals, best = self.best_values(v, val)
            g = cst - best
            cost[v], improve[v] = cst, g
            if self._improving(g):
                _, w = philox.draw(self.seed, self.var_id[v], cyc)
                new_value[v] = vals[philox.choice_index(w, len(vals))]
                self.stats["multi_draws"] += len(vals) >= 2
        # improve phase (:493-541): the breakouts read this round's values
        new_val, breakout = list(val), [False] * V
        for v in conn:
            mine = improve[v]
            maxi, tied = mine, [self.rank[v]]
            for u in self.nbrs[v]:
                if improve[u] > maxi:
                    maxi, tied = improve[u], [self.rank[u]]
                elif improve[u] == maxi:
                    tied.append(self.rank[u])
            if self._improving(mine):
                if mine == maxi and len(tied) > 1:
                    self.stats["rank_decided"] += 1
                if min(tied) == self.rank[v]:
                    new_val[v] = new_value[v]
                    cost[v] = cost[v] + mine
            elif maxi == 0:
                hit = [k for k in range(len(self.cons[v])) if violated[v][k]]
                for k in hit:
                    self.increase_cost(v, k, val)
                    if self.increase_mode != "T":
                        if self.span[v][k]:
                            self.stats["span_increases"] += 1
                        else:
                            self.stats["other_breakout_slots"] += 1
                if hit:
                    breakout[v] = True
                    self.stats["breakouts"] += 1
                    if self.mode_max and any(self._improving(improve[u]) for u in self.nbrs[v]):
                        self.stats["max_breakouts_next_to_improving"] += 1
        self.val, self.cost = new_val, cost
        self.last = dict(improve=improve, new_value=new_value, violated=violated, breakout=breakout)

    # -- views -----------------------------------------------------------------------------------
    def values(self):
        """(value index per variable, current cost or NaN while the reference's is None)."""
        cost = np.array([np.nan if c is None else float(c) for c in self.cost])
        return np.array(self.val, dtype=np.int32), cost

    def modifiers(self):
        """Every modifier as the reads see it: per variable, per slot (node.constraints order), the
        constraint's entries in table order, flattened."""
        out = []
        for v in range(self.V):
            for k, f in enumerate(self.cons[v]):
                out.append(np.array([self.modifier_at(v, k, i) for i in range(self.tsize[f])], dtype=np.int32))
        return np.concatenate(out) if out else np.zeros(0, np.int32)

    def record(self):
        """The per-round fixture arrays of the last round (NaN / -1 / 0 without neighbours)."""
        L = self.last
        conn = np.array([bool(n) for n in self.nbrs])
        return dict(improve=np.array([float(g) if conn[v] else np.nan for v, g in enumerate(L["improve"])]),
                    new_value=np.where(conn, np.array(L["new_value"]), -1).astype(np.int32),
                    violated=np.array([x for row in L["violated"] for x in row], dtype=np.uint8),
                    breakout=np.array(L["breakout"], dtype=np.uint8),
                    modifiers=self.modifiers())
