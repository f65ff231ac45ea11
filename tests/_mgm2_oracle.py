"""MGM-2 restated in plain Python: the oracle of the `mgm2_*` fixtures and of the MGM-2 kernels.
TEST INFRASTRUCTURE ONLY (the product package never imports it).

One `step()` is one MGM-2 cycle of pydcop/algorithms/mgm2.py for every variable at once, in the
reference's arithmetic: every cost is a sum from 0 over the variable's constraints in
`node.constraints` order (`assignment_cost`, relations.py:1479-1532, without variable costs), in
the precision of `dtype` (np.float32 scalars round every operation to f32).

Random draws are injected: Philox4x32-10 with counter (canonical variable id, cycle, purpose, 0)
(`draw`), cycle = 0xffffffff for the start values, else the variable's 1-based round.  Purposes:
0 start value, 1 offerer coin (u) and partner pick (choice word), 2 unilateral value pick,
3 `favor="no"` coin, 4 offer pick.  Lists are indexed in canonical order: neighbours in order of
first appearance over the variable's constraints, then scope order; best values in domain order;
best offers by (offerer's neighbour position, offerer value, own value).
"""
import numpy as np

import philox

PURPOSE_INIT, PURPOSE_OFFER, PURPOSE_VALUE, PURPOSE_FAVOR, PURPOSE_PICK = 0, 1, 2, 3, 4
FAVORS = ("unilateral", "no", "coordinated")


def draw(seed: int, var: int, cycle: int, purpose: int):
    """(u in [0, 1), choice word) of Philox counter (var, cycle, purpose, 0); purpose 0 is
    oracle/philox.py's `draw`."""
    b = philox.philox4x32_10((var, cycle, purpose, 0), (seed & philox.MASK, (seed >> 32) & philox.MASK))
    u = ((b[0] >> 5) * 67108864 + (b[1] >> 6)) / 9007199254740992.0
    return u, b[2]


def neighbour_lists(dom_size, factor_ptr, edge_var, var_ptr, var_con):
    """Distinct neighbours of every variable in first-appearance order (canonical ids)."""
    out = []
    for v in range(len(dom_size)):
        seen = []
        for s in range(var_ptr[v], var_ptr[v + 1]):
            f = var_con[s]
            for u in edge_var[factor_ptr[f]:factor_ptr[f + 1]]:
                u = int(u)
                if u != v and u not in seen:
                    seen.append(u)
        out.append(seen)
    return out


def var_constraints(inst):
    """Constraint id of every slot (fixtures carry var_con, engine instances var_edge)."""
    if "var_con" in inst:
        return np.asarray(inst["var_con"], dtype=np.int64)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    fac = np.repeat(np.arange(len(fp) - 1), np.diff(fp))
    return fac[np.asarray(inst["var_edge"], dtype=np.int64)]


class Mgm2Oracle:
    """Lock-step MGM-2.  State after `init()` == fixture row 0, after n `step()` == row n."""

    def __init__(self, inst, dtype=np.float64, mode="min", threshold=0.5, favor="unilateral",
                 stop_cycle=0, seed=0, var_id=None, **_ignored):
        if favor not in FAVORS:
            raise ValueError(f"invalid favor {favor!r}")
        self.T = np.float64 if np.dtype(dtype) == np.float64 else np.float32
        self.mode_max = mode == "max"
        self.threshold, self.favor = float(threshold), favor
        self.stop_cycle, self.seed = int(stop_cycle or 0), int(seed)
        self.dom = [int(x) for x in inst["dom_size"]]
        V = self.V = len(self.dom)
        fp = [int(x) for x in inst["factor_ptr"]]
        ev = [int(x) for x in inst["edge_var"]]
        if "table_off" in inst and inst["table_off"] is not None:
            toff = [int(x) for x in inst["table_off"]]
        else:
            toff = [0]
            for f in range(len(fp) - 1):
                toff.append(toff[-1] + int(np.prod([self.dom[u] for u in ev[fp[f]:fp[f + 1]]])))
        self.tables = np.ascontiguousarray(inst["tables"], dtype=self.T)
        self.scope = [ev[fp[f]:fp[f + 1]] for f in range(len(fp) - 1)]
        self.toff = toff
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
        iv = inst["init_value"] if "init_value" in inst else None
        self.init_value = [int(x) for x in iv] if iv is not None else [-1] * V
        rank = inst["var_rank"] if "var_rank" in inst else None
        self.rank = [int(x) for x in rank] if rank is not None else list(range(V))
        self.var_id = [int(x) for x in var_id] if var_id is not None else list(range(V))
        self.cycle = 0

    # -- costs -----------------------------------------------------------------------------
    def _cost(self, fs, val):
        """assignment_cost: 0 + c_1 + c_2 + ... over the constraints `fs` at assignment `val`."""
        c = self.T(0)
        for f in fs:
            i = self.toff[f]
            for u, s in zip(self.scope[f], self.strides[f]):
                i += val[u] * s
            c = c + self.tables[i]
        return c

    def _better(self, a, b):
        """a strictly better than b (the reference's `a < b` in min mode, `a > b` in max mode)."""
        return a > b if self.mode_max else a < b

    def _best_values(self, v, val):
        """_compute_best_value (mgm2.py:495-519): (best values in domain order, best cost)."""
        work = list(val)
        best, vals = None, []
        for x in range(self.dom[v]):
            work[v] = x
            c = self._cost(self.cons[v], work)
            if best is None or self._better(c, best):
                best, vals = c, [x]
            elif c == best:
                vals.append(x)
        return vals, best

    # -- lifecycle -------------------------------------------------------------------------
    def init(self):
        V = self.V
        self.val = [0] * V
        self.cost = [None] * V
        self.is_finished = [False] * V
        for v in range(V):
            if self.nbrs[v]:
                if self.init_value[v] >= 0:
                    self.val[v] = self.init_value[v]
                else:
                    _, w = draw(self.seed, self.var_id[v], philox.INIT_CYCLE, PURPOSE_INIT)
                    self.val[v] = philox.choice_index(w, self.dom[v])
            else:  # on_start without neighbours (mgm2.py:465-475)
                vals, best = self._best_values(v, self.val)
                _, w = draw(self.seed, self.var_id[v], philox.INIT_CYCLE, PURPOSE_INIT)
                self.val[v] = vals[philox.choice_index(w, len(vals))]
                self.cost[v] = best
                self.is_finished[v] = True
        self.cycle = 0
        self.last = None
        # how often the favor rule decided (best offer gain == unilateral gain != 0), and how
        self.stats = dict(ties=0, tie_commits=0, coin_commit=0, coin_refuse=0)
        return self

    @property
    def finished(self):
        """_send_value (mgm2.py:605-622): cycle_count (= rounds done + 1) reached stop_cycle."""
        return bool(self.stop_cycle and self.cycle + 1 >= self.stop_cycle)

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self._round(self.cycle + 1)
            self.cycle += 1
        return self

    def _round(self, cyc):
        T, V, seed = self.T, self.V, self.seed
        zero = T(0)
        val = self.val
        conn = [v for v in range(V) if self.nbrs[v]]
        local = [None] * V
        offerer = [False] * V
        partner = [-1] * V          # canonical id
        pgain = [zero] * V
        pvalue = list(val)
        committed = [False] * V
        offers = {}
        # 1. value phase: current cost, unilateral move, offerer coin, offer table (mgm2.py:742-785)
        for v in conn:
            cst = self._cost(self.cons[v], val)
            local[v] = cst
            u, w = draw(seed, self.var_id[v], cyc, PURPOSE_OFFER)
            if u < self.threshold:
                offerer[v] = True
                p = self.nbrs[v][philox.choice_index(w, len(self.nbrs[v]))]
                partner[v] = p
                work, table = list(val), {}
                for a in range(self.dom[v]):       # generate_assignment_as_dict([self, partner])
                    work[v] = a
                    for b in range(self.dom[p]):
                        work[p] = b
                        c = self._cost(self.cons[v], work)
                        if self._better(c, cst):
                            table[(a, b)] = cst - c
                offers[v] = table
            vals, best = self._best_values(v, val)
            g = cst - best
            pgain[v] = g
            if (g < 0) if self.mode_max else (g > 0):
                _, w = draw(seed, self.var_id[v], cyc, PURPOSE_VALUE)
                pvalue[v] = vals[philox.choice_index(w, len(vals))]
        # 2. answers of the receivers (mgm2.py:787-856, _find_best_offer :556-603)
        accepted = {}
        for v in conn:
            if offerer[v]:
                continue
            bests, best = [], zero
            work = list(val)
            for u in self.nbrs[v]:
                if not offerer[u] or partner[u] != v:
                    continue
                concerned = [f for f in self.cons[v] if u not in self.scope[f]]
                for (a, b), pg in offers[u].items():
                    work[v] = b
                    gg = (local[v] - self._cost(concerned, work)) + pg
                    if (gg < best) if self.mode_max else (gg > best):
                        bests, best = [(u, a, b)], gg
                    elif gg == best:
                        bests.append((u, a, b))
            commit = False
            if best == 0 or not bests:
                commit = False
            elif (best < pgain[v]) if self.mode_max else (best > pgain[v]):
                commit = True
            elif best == pgain[v]:
                self.stats["ties"] += 1
                if self.favor == "coordinated":
                    commit = True
                elif self.favor == "no":
                    u3, _ = draw(seed, self.var_id[v], cyc, PURPOSE_FAVOR)
                    commit = u3 > 0.5
                    self.stats["coin_commit" if commit else "coin_refuse"] += 1
                if commit:
                    self.stats["tie_commits"] += 1
            if commit:
                _, w = draw(seed, self.var_id[v], cyc, PURPOSE_PICK)
                u, a, b = bests[philox.choice_index(w, len(bests))]
                committed[v], pgain[v], pvalue[v], partner[v] = True, best, b, u
                accepted[u] = (a, best)
        # 3. offerers read their answer (mgm2.py:858-890)
        for u, (a, g) in accepted.items():
            committed[u], pvalue[u], pgain[u] = True, a, g
        # 4. gain phase (mgm2.py:892-972)
        go = [False] * V
        new_val, new_cost = list(val), [local[v] if local[v] is not None else self.cost[v] for v in range(V)]
        for v in conn:
            g = pgain[v]
            if g == 0:
                continue
            if committed[v]:
                others = [pgain[u] for u in self.nbrs[v] if u != partner[v]]
                go[v] = not others or g > max(others)
                continue
            mx = max(pgain[u] for u in self.nbrs[v])
            move = False
            if g > mx:
                move = True
            elif g == mx:
                move = all(not (pgain[u] == mx and self.rank[u] < self.rank[v]) for u in self.nbrs[v])
            if move:
                new_val[v], new_cost[v] = pvalue[v], local[v] - g
        # 5. coordinated moves (mgm2.py:974-1001)
        for v in conn:
            if committed[v] and go[v] and go[partner[v]]:
                new_val[v], new_cost[v] = pvalue[v], local[v] - pgain[v]
        self.val, self.cost = new_val, new_cost
        pos = [self.nbrs[v].index(partner[v]) if partner[v] >= 0 else -1 for v in range(V)]
        self.last = dict(local_cost=local, offerer=offerer, partner=pos, committed=committed,
                         gain=pgain, potential_value=pvalue, go=go)

    # -- views -----------------------------------------------------------------------------
    def values(self):
        """(value index per variable, current cost or NaN while the reference's is None)."""
        cost = np.array([np.nan if c is None else float(c) for c in self.cost])
        return np.array(self.val, dtype=np.int32), cost

    def record(self):
        """The per-cycle fixture arrays of the last round, NaN / -1 / 0 where a variable has none."""
        V, L = self.V, self.last
        conn = np.array([bool(n) for n in self.nbrs])
        f = lambda xs: np.array([np.nan if (x is None or not conn[i]) else float(x)  # noqa: E731
                                 for i, x in enumerate(xs)])
        return dict(local_cost=f(L["local_cost"]), offerer=np.array(L["offerer"], dtype=np.uint8),
                    partner=np.array(L["partner"], dtype=np.int32),
                    committed=np.array(L["committed"], dtype=np.uint8), gain=f(L["gain"]),
                    potential_value=np.where(conn, np.array(L["potential_value"]), -1).astype(np.int32),
                    go=np.array(L["go"], dtype=np.uint8))
