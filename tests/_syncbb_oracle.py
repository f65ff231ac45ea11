"""Python restatement of the reference SyncBB (pydcop/algorithms/syncbb.py:176-512) for the tests, one message per
`step()`, in float64 or float32 (every cost, bound and sum in that precision).

The chain is the variables sorted by name (ordered_graph.py:173, `var_rank`); the path is always a prefix of the
chain, so path element q belongs to the variable at chain position q.  Per candidate and path element (u, val_u,
elt_cost) in path order, `ass` is the sum, from 0 in node.constraints order, of v's binary constraints on u at
(val_u, candidate); a min-mode element fails when `cc + ass >= ub or ass + elt_cost >= ub`; a candidate is rejected
only when its FIRST element fails, otherwise accepted with the cost summed up to the last element that passed
(:448-473).  Max mode accepts every candidate with its full sum.  Unary constraints and variable costs are never read.
"""
import numpy as np

FORWARD, BACKWARD, TERMINATE = 0, 1, 2


def table_offsets(inst):
    if "table_off" in inst:
        return np.asarray(inst["table_off"], dtype=np.int64)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"], dtype=np.int64)
    sizes = [int(np.prod(dom[ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)]
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def slot_constraints(inst):
    """node.constraints of every variable: fixtures carry var_con, engine instances var_edge (or neither: the
    constraints in canonical order)."""
    V = len(inst["dom_size"])
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    if "var_con" in inst:
        vp, vc = np.asarray(inst["var_ptr"]), np.asarray(inst["var_con"])
    elif "var_edge" in inst:
        fac = np.repeat(np.arange(len(fp) - 1), np.diff(fp))
        vp, vc = np.asarray(inst["var_ptr"]), fac[np.asarray(inst["var_edge"], dtype=np.int64)]
    else:
        ev = np.asarray(inst["edge_var"], dtype=np.int64)
        out = [[] for _ in range(V)]
        for f in range(len(fp) - 1):
            for v in dict.fromkeys(int(x) for x in ev[fp[f]:fp[f + 1]]):
                out[v].append(f)
        return out
    return [[int(x) for x in vc[vp[v]:vp[v + 1]]] for v in range(V)]


def python_sum(xs, dt):
    """`sum()` of Python floats as CPython 3.12 computes it (Neumaier's compensated summation, the compensation
    added at the end only when it is finite and non-zero), in precision `dt`.  syncbb.py:290 sums the path's costs
    with it."""
    f, c = dt(0), dt(0)
    for x in xs:
        x = dt(x)
        t = dt(f + x)
        if abs(f) >= abs(x):
            c = dt(c + dt(dt(f - t) + x))
        else:
            c = dt(c + dt(dt(x - t) + f))
        f = t
    return dt(f + c) if c != 0 and np.isfinite(c) else f


class SyncbbOracle:
    def __init__(self, inst, dtype=np.float64, mode="min", var_rank=None):
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        self.dt, self.mode = dtype, mode
        dom = np.asarray(inst["dom_size"], dtype=np.int64)
        V = self.n = len(dom)
        fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
        ev = np.asarray(inst["edge_var"], dtype=np.int64)
        toff = table_offsets(inst)
        tables = np.asarray(inst["tables"], dtype=np.float64).astype(dtype)
        rank = np.arange(V) if var_rank is None else np.asarray(var_rank, dtype=np.int64)
        self.chain = np.argsort(rank, kind="stable")      # chain position -> canonical variable
        self.pos = np.empty(V, dtype=np.int64)
        self.pos[self.chain] = np.arange(V)
        self.dom = dom[self.chain]
        # ass[p] = {q: table [val_u][x]} for every earlier u (position q) sharing a constraint with chain position p
        self.ass = [dict() for _ in range(V)]
        for v, cons in enumerate(slot_constraints(inst)):
            p = int(self.pos[v])
            for f in cons:
                scope = [int(x) for x in ev[fp[f]:fp[f + 1]]]
                if len(scope) > 2:
                    raise ValueError(f"constraint {f} has arity {len(scope)}: SyncBB supports binary constraints only")
                if len(scope) < 2:
                    continue
                u = scope[0] if scope[1] == v else scope[1]
                q = int(self.pos[u])
                if q >= p:
                    continue
                t = tables[toff[f]:toff[f + 1]].reshape(int(dom[scope[0]]), int(dom[scope[1]]))
                t = t if scope[0] == u else t.T
                self.ass[p][q] = (self.ass[p].get(q, dtype(0)) + t).astype(dtype)

    # ---- state ----------------------------------------------------------------------------------------------
    def init(self):
        V, dt = self.n, self.dt
        if V < 2:
            raise ValueError("SyncBB needs at least two variables")
        self.inf = dt(np.inf) if self.mode == "min" else dt(-np.inf)
        self.ub = np.full(V, self.inf, dtype=dt)
        self.sel = np.full(V, -1, dtype=np.int32)
        self.path_val = np.zeros(V, dtype=np.int32)
        self.path_cost = np.zeros(V, dtype=dt)
        self.msg = (FORWARD, 1, 1, self.inf)       # syncbb.py:205-210: [(x0, domain[0], 0)], bound +-inf
        self.steps, self.messages, self.finished = 0, 1, False
        self.cycles = np.zeros(V, dtype=np.int64)        # new_cycle count per variable: on_start (:211), then
        self.cycles[0] = 1                               # one per message handled
        self.stats = dict(partial=0, rejected=0, pruned_by_inf=0, improved=0)
        return self

    def _next(self, p, start, plen, ub):
        """get_next_assignment (:415-473) at chain position p for candidates start.. against the path prefix of
        length plen: (value, cost) or None."""
        dt = self.dt
        for x in range(start, int(self.dom[p])):
            if plen == 0:
                return x, dt(0)
            cc, found = dt(0), None
            for q in range(plen):
                t = self.ass[p].get(q)
                a = t[self.path_val[q], x] if t is not None else dt(0)
                c2 = dt(cc + a)
                if self.mode == "min" and (c2 >= ub or dt(a + self.path_cost[q]) >= ub):
                    if q > 0:
                        self.stats["partial"] += 1
                    elif np.isinf(ub) and ub > 0:
                        self.stats["pruned_by_inf"] += 1
                    break
                cc, found = c2, (x, c2)
            if found is not None:
                return found
            self.stats["rejected"] += 1
        return None

    def _post(self, kind, to, plen, ub):
        self.messages += 1
        self.msg = (kind, to, plen, ub)

    def step(self):
        """Deliver the message in flight; returns False once finished."""
        if self.finished:
            return False
        kind, p, plen, mub = self.msg
        n, dt = self.n, self.dt
        self.steps += 1
        self.cycles[p] += 1
        better = (lambda a, b: a < b) if self.mode == "min" else (lambda a, b: a > b)
        if kind == TERMINATE:                        # :213-232
            if p + 1 < n:
                self._post(TERMINATE, p + 1, 0, dt(np.nan))
            else:
                self.finished = True
            return True
        if kind == FORWARD:                          # :234-341, the forward ub is ignored (:248)
            nxt = self._next(p, 0, plen, self.ub[p])
            if nxt is None:
                self._post(BACKWARD, p - 1, plen, self.ub[p])       # the root never receives forward
            elif p == n - 1:                        # :287-328
                bound = python_sum(self.path_cost[:plen], dt)
                best_val, best = None, self.ub[p]
                while nxt is not None:
                    x, c = nxt
                    if better(dt(bound + c), best):
                        best, best_val = dt(bound + c), x
                    nxt = self._next(p, x + 1, plen, self.ub[p])
                if best_val is not None:
                    self.ub[p] = best
                    self.sel[p] = best_val
                    self.stats["improved"] += 1
                self._post(BACKWARD, p - 1, plen, self.ub[p])
            else:
                x, c = nxt
                self.path_val[p], self.path_cost[p] = x, c
                self._post(FORWARD, p + 1, p + 1, self.ub[p])
            return True
        # BACKWARD (:343-412): the last path element is the receiver's own
        val = int(self.path_val[p])
        if better(mub, self.ub[p]):
            self.ub[p] = mub
            self.sel[p] = val
        nxt = self._next(p, val + 1, p, self.ub[p])
        if nxt is not None:
            x, c = nxt
            self.path_val[p], self.path_cost[p] = x, c
            self._post(FORWARD, p + 1, p + 1, self.ub[p])
        elif p == 0:
            self._post(TERMINATE, 1, 0, dt(np.nan))
        else:
            self._post(BACKWARD, p - 1, p, self.ub[p])
        return True

    def run(self, max_steps=None):
        k = 0
        while not self.finished and (max_steps is None or k < max_steps):
            self.step()
            k += 1
        return self

    # ---- readers, canonical order -----------------------------------------------------------------------------
    def canonical(self, a):
        out = np.empty_like(a)
        out[self.chain] = a
        return out

    def values(self):
        """Last value_selection per variable, -1 for a variable that never selected."""
        return self.canonical(self.sel)

    def bounds(self):
        return self.canonical(self.ub)

    def cycle_counts(self):
        """Each variable's new_cycle count; the orchestrator reports the largest as the run's `cycle`."""
        return self.canonical(self.cycles)

    def message(self):
        """The message in flight: (type, receiver as canonical index, path length, bound carried)."""
        kind, p, plen, ub = self.msg
        return kind, int(self.chain[p]), plen, ub
