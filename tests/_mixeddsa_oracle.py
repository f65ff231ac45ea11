"""MixedDSA restated in plain Python: the oracle of the `mixeddsa_*` fixtures and of the MixedDSA kernel.
TEST INFRASTRUCTURE ONLY (the product package never imports it).

One `step()` is one lock-step round of pydcop/algorithms/mixeddsa.py (MixedDsaComputation._on_neighbors_values
:272-373) for every variable at once, in the precision of `dtype` (np.float32 scalars round every operation to f32).

Classification (:205-225): a constraint is hard iff its table, in `dtype`, holds +inf or -inf; its optimum is the
table's min (max in max mode), kept for the soft ones.

Cost of a candidate x (_compute_dcop_cost :410-446), the neighbours at their values of the previous round:
  C(x) = ((0 + soft_1 + soft_2 + ...) + own cost at x + the neighbours' costs) + every hard entry that is not +inf
  H(x) = number of hard entries equal to +inf
Soft and hard constraints each in node.constraints order.  The variable costs are those of `concerned_vars`, a set
the reference sums in hash order: here own first, then the neighbours in order of first appearance (the fixtures
use integer or dyadic costs, for which every order gives the same sum).  A variable without constraints has none.

Best values (_compute_best_value :381-402), decision (:300-358) and reported cost (_eff_cost :448-462) as the
reference reads; variant C takes variant B's branch (:342 is unreachable).  A variable without neighbours evaluates
once, in round 1 (it does so from on_start in the reference, with cycle_count 1, and then never again).

Random draws are injected as DSA's: Philox4x32-10 with counter (canonical variable id, cycle, 0, 0)
(oracle/philox.py `draw`): u for the probability test and the choice index from the same block, cycle = the
1-based round; cycle 0xffffffff for the start value of every variable without an initial value.

Branch codes (fg_mixeddsa_desc_t dev_branch): 1 dH > 0, 2 soft improvement, 3 stuck with violated hard
constraints, 4 stuck on a violated soft constraint (B / C), 5 none of them, 0 no evaluation; + 8 when the
variable moved.
"""
import numpy as np

import philox
from _mgm2_oracle import neighbour_lists, var_constraints

VARIANTS = ("A", "B", "C")
BRANCH_NONE, BRANCH_HARD, BRANCH_SOFT, BRANCH_STUCK_HARD, BRANCH_STUCK_SOFT, BRANCH_IDLE = range(6)
MOVED = 8


class MixedDsaOracle:
    """Lock-step MixedDSA.  State after `init()` == fixture row 0, after n `step()` == row n."""

    def __init__(self, inst, dtype=np.float64, mode="min", proba_hard=0.7, proba_soft=0.5, variant="B",
                 stop_cycle=0, seed=0, var_id=None, **_ignored):
        if variant not in VARIANTS:
            raise ValueError(f"invalid variant {variant!r}")
        self.T = np.float64 if np.dtype(dtype) == np.float64 else np.float32
        self.mode_max = mode == "max"
        self.proba_hard, self.proba_soft, self.variant = float(proba_hard), float(proba_soft), variant
        self.stop_cycle, self.seed = int(stop_cycle or 0), int(seed)
        self.dom = [int(x) for x in inst["dom_size"]]
        V = self.V = len(self.dom)
        fp = [int(x) for x in inst["factor_ptr"]]
        ev = [int(x) for x in inst["edge_var"]]
        tsize = [int(np.prod([self.dom[u] for u in ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)]
        toff = [0] + [int(x) for x in np.cumsum(tsize, dtype=np.int64)]
        if "table_off" in inst and inst["table_off"] is not None:
            toff = [int(x) for x in inst["table_off"]]
        tables = np.ascontiguousarray(inst["tables"], dtype=self.T)
        self.table = [tables[toff[f]:toff[f] + tsize[f]] for f in range(len(tsize))]
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
        self.hard = [bool(np.isinf(t).any()) for t in self.table]
        self.opt = []
        for t in self.table:   # strict comparison from the first entry (:211-218)
            o = t[0] if len(t) else None
            for x in t[1:]:
                if (x > o) if self.mode_max else (x < o):
                    o = x
            self.opt.append(o)
        self.soft_cons = [[f for f in self.cons[v] if not self.hard[f]] for v in range(V)]
        self.hard_cons = [[f for f in self.cons[v] if self.hard[f]] for v in range(V)]
        uoff = np.concatenate([[0], np.cumsum(self.dom)]).astype(np.int64)
        unary = np.asarray(inst["unary"], dtype=self.T) if "unary" in inst else np.zeros(int(uoff[-1]), self.T)
        self.unary = [unary[uoff[v]:uoff[v + 1]] for v in range(V)]
        iv = inst["init_value"] if "init_value" in inst else None
        self.init_value = [int(x) for x in iv] if iv is not None else [-1] * V
        self.var_id = [int(x) for x in var_id] if var_id is not None else list(range(V))
        self.cycle = 0

    def _entry(self, f, val):
        return self.table[f][sum(val[u] * s for u, s in zip(self.scope[f], self.strides[f]))]

    def dcop_cost(self, v, val):
        """_compute_dcop_cost with the assignment `val`: (C, H)."""
        acc = self.T(0)
        for f in self.soft_cons[v]:
            acc = acc + self._entry(f, val)
        if self.cons[v]:
            acc = acc + self.unary[v][val[v]]
            for u in self.nbrs[v]:
                acc = acc + self.unary[u][val[u]]
        h = 0
        for f in self.hard_cons[v]:
            e = self._entry(f, val)
            if e == np.inf:
                h += 1
            else:
                acc = acc + e
        return acc, h

    def best_values(self, v, val):
        """_compute_best_value: (H_best, C_best, bests in domain order)."""
        work = list(val)
        best_c, best_h, bests = None, len(self.hard_cons[v]) + 1, []
        for x in range(self.dom[v]):
            work[v] = x
            c, h = self.dcop_cost(v, work)
            if h < best_h:
                best_c, best_h, bests = c, h, [x]
            elif h == best_h:
                if (c > best_c) if self.mode_max else (c < best_c):
                    best_c, bests = c, [x]
                elif c == best_c:
                    bests.append(x)
        return best_h, best_c, bests

    def soft_violated(self, v, val):
        """exists_violated_soft_constraint (:464-476), the function-relation meaning."""
        return any(self._entry(f, val) != self.opt[f] for f in self.soft_cons[v])

    # -- lifecycle -----------------------------------------------------------------------------
    def init(self):
        self.val, self.cost = [0] * self.V, [None] * self.V
        for v in range(self.V):
            if self.init_value[v] >= 0:
                self.val[v] = self.init_value[v]
            else:
                _, w = philox.draw(self.seed, self.var_id[v], philox.INIT_CYCLE)
                self.val[v] = philox.choice_index(w, self.dom[v])
        self.cycle = 0
        self.last = None
        return self

    @property
    def finished(self):
        """stop_cycle with dsa_gpu's convention: the run ends after stop_cycle rounds."""
        return bool(self.stop_cycle and self.cycle >= self.stop_cycle)

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self._round(self.cycle + 1)
            self.cycle += 1
        return self

    def decide(self, v, val, cyc):
        """One evaluation of v: (new value, eff_cost or None without a move, H_best, branch code)."""
        cur = val[v]
        h_best, c_best, bests = self.best_values(v, val)
        c_cur, h_cur = self.dcop_cost(v, val)
        with np.errstate(invalid="ignore"):    # inf - inf: NaN, as in Python
            dh, dc = h_cur - h_best, c_cur - c_best
        u, w = philox.draw(self.seed, self.var_id[v], cyc)
        eff = self.T(np.inf) if h_best else c_best
        br, p, drop = BRANCH_IDLE, None, False
        if dh > 0:
            br, p = BRANCH_HARD, self.proba_hard
        elif dh == 0:
            if (dc < 0) if self.mode_max else (dc > 0):
                br, p = BRANCH_SOFT, self.proba_soft
            elif dc == 0:
                if h_best > 0:
                    br, drop = BRANCH_STUCK_HARD, True
                    p = self.proba_hard if len(bests) > 1 else None
                elif self.soft_violated(v, val) and self.variant in ("B", "C"):
                    br, drop = BRANCH_STUCK_SOFT, True
                    p = self.proba_soft if len(bests) > 1 else None
        if p is not None and p > u:
            if drop:
                bests = [x for x in bests if x != cur]
            return bests[philox.choice_index(w, len(bests))], eff, h_best, br | MOVED
        return cur, None, h_best, br

    def _round(self, cyc):
        val = self.val
        new_val, cost = list(val), list(self.cost)
        h_best, branch = [-1] * self.V, [BRANCH_NONE] * self.V
        for v in range(self.V):
            if not self.nbrs[v] and cyc != 1:
                continue
            nv, eff, h_best[v], branch[v] = self.decide(v, val, cyc)
            if branch[v] & MOVED:
                new_val[v], cost[v] = nv, eff
        self.val, self.cost = new_val, cost
        self.last = dict(h_best=np.array(h_best, dtype=np.int32), branch=np.array(branch, dtype=np.uint8))

    # -- views -----------------------------------------------------------------------------------
    def values(self):
        """(value index per variable, current cost or NaN while the reference's is None)."""
        cost = np.array([np.nan if c is None else float(c) for c in self.cost])
        return np.array(self.val, dtype=np.int32), cost

    def record(self):
        """h_best and branch of the last round per variable."""
        return dict(self.last)
