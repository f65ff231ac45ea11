"""Vectorised numpy restatement of DPOP (pydcop/algorithms/dpop.py:115-441) in the engine's fixed
summation order, the CPU oracle of csrc/dpop_kernels.cuh.

A node's joined table, axes [own variable] + separator (root side first), is the left-associated sum,
in the oracle's dtype, of its own cost row, each child's UTIL (children order) and each constraint it
owns (constraint order).  The UTIL sent up is its projection over the own axis with the reference's
find_arg_optimal: the running best starts at the int32 sentinel (2147483647 in min mode, -2147483648 in
max mode; in f32 the sentinel rounds to 2^31) and only a strictly better entry replaces it, so NaN never
wins.  VALUE recomputes the one joined row at the separator's values; the value is the first index whose
entry equals the best, and where none does (the reference raises IndexError) the oracle, like the engine,
takes value 0 and cost NaN and counts the node as unresolved.
"""
import numpy as np


def sentinel(dt, mode):
    return dt(-2147483648.0) if mode == "max" else dt(2147483647.0)


def _expand(arr, arr_vars, target_vars):
    """`arr` (axes arr_vars) as a view broadcastable over the axes target_vars."""
    pos = {v: i for i, v in enumerate(target_vars)}
    perm = sorted(range(len(arr_vars)), key=lambda i: pos[arr_vars[i]])
    a = arr.transpose(perm)
    shape = [1] * len(target_vars)
    for i in perm:
        shape[pos[arr_vars[i]]] = arr.shape[i]
    return a.reshape(shape)


class DpopOracle:
    def __init__(self, inst, tree, dt=np.float64, mode="min"):
        self.dt, self.mode, self.tree = dt, mode, tree
        self.dom = np.asarray(inst["dom_size"], dtype=np.int64)
        fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
        ev = np.asarray(inst["edge_var"], dtype=np.int64)
        tables = np.asarray(inst["tables"], dtype=np.float64)
        toff = inst.get("table_off") if hasattr(inst, "get") else None
        if toff is None:
            sizes = [int(np.prod(self.dom[ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)]
            toff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        V = len(self.dom)
        self.scopes = [ev[fp[f]:fp[f + 1]].tolist() for f in range(len(fp) - 1)]
        self.tables = [tables[toff[f]:toff[f + 1]].astype(dt).reshape(tuple(self.dom[s]))
                       for f, s in enumerate(self.scopes)]
        un = inst.get("unary") if hasattr(inst, "get") else None
        uoff = np.concatenate([[0], np.cumsum(self.dom)])
        un = np.zeros(int(uoff[-1])) if un is None else np.asarray(un, dtype=np.float64)
        self.unary = [un[uoff[v]:uoff[v + 1]].astype(dt) for v in range(V)]
        self.owned = tree.owned
        self.util = [None] * V
        self.value = np.zeros(V, dtype=np.int32)
        self.cost = np.full(V, np.nan)
        self.unresolved = 0

    def _better(self, e, best):
        return e > best if self.mode == "max" else e < best

    def joined(self, u):
        axes = [u] + self.tree.sep[u]
        shape = tuple(int(self.dom[v]) for v in axes)
        j = np.broadcast_to(_expand(self.unary[u], [u], axes), shape).copy()
        for c in self.tree.children[u]:
            j = j + _expand(self.util[c], self.tree.sep[c], axes)
        for f in self.owned[u]:
            j = j + _expand(self.tables[f], self.scopes[f], axes)
        return j.astype(self.dt, copy=False)

    def util_phase(self):
        for u in reversed(self.tree.preorder()):
            j = self.joined(u)
            best = np.full(j.shape[1:], sentinel(self.dt, self.mode), dtype=self.dt)
            for v in range(j.shape[0]):
                upd = self._better(j[v], best)
                best = np.where(upd, j[v], best)
            self.util[u] = best
        return self

    def row(self, u):
        """The joined row of u at its separator's chosen values, same operand order."""
        val = {v: int(self.value[v]) for v in self.tree.sep[u]}
        r = self.unary[u].copy()

        def sl(scope):
            return tuple(slice(None) if w == u else val[w] for w in scope)
        for c in self.tree.children[u]:
            r = r + self.util[c][sl(self.tree.sep[c])]
        for f in self.owned[u]:
            r = r + self.tables[f][sl(self.scopes[f])]
        return r.astype(self.dt, copy=False)

    def value_phase(self):
        for u in self.tree.preorder():
            best, arg = sentinel(self.dt, self.mode), -1
            for v, e in enumerate(self.row(u)):
                if self._better(e, best):
                    best, arg = e, v
                elif e == best and arg < 0:
                    arg = v
            if arg < 0:
                self.value[u], self.cost[u] = 0, np.nan
                self.unresolved += 1
            else:
                self.value[u], self.cost[u] = arg, float(best)
        return self

    def run(self):
        return self.util_phase().value_phase()

    def values(self):
        return self.value, self.cost


def brute_force(inst, mode="min"):
    """Optimal total cost over every assignment (constraints + variable costs), f64."""
    import itertools
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"], dtype=np.int64)
    tables = np.asarray(inst["tables"], dtype=np.float64)
    toff = np.concatenate([[0], np.cumsum([int(np.prod(dom[ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)])])
    uoff = np.concatenate([[0], np.cumsum(dom)])
    un = np.asarray(inst.get("unary", np.zeros(int(uoff[-1]))), dtype=np.float64)
    best = None
    for a in itertools.product(*[range(int(d)) for d in dom]):
        c = sum(un[uoff[v] + x] for v, x in enumerate(a))
        for f in range(len(fp) - 1):
            s = ev[fp[f]:fp[f + 1]]
            c += tables[toff[f] + int(np.ravel_multi_index(tuple(a[v] for v in s), tuple(dom[s])))]
        if best is None or (c > best if mode == "max" else c < best):
            best = c
    return best
