"""DBA restated in plain Python: the oracle of the `dba_*` fixtures and of the DBA kernels.
TEST INFRASTRUCTURE ONLY (the product package never imports it).

One `step()` is one round of pydcop/algorithms/dba.py for every variable at once, under lock-step delivery: the
ok phase (:366-420) of every variable, then its improve phase (:504-562).  Phases are numbered p = 2k (ok) and
2k + 1 (improve) for round k = 1, 2, ...

  eval(x)   = sum of weight[k] over the slots k (node.constraints order) whose entry at x is >= infinity,
              compared in the tables' precision (`dtype`)
  best      = strict minimum starting from `infinity`, ties in domain order; improve = eval(cur) - best
  End flood = a live variable finishes at phase p iff a neighbour finished at a phase < p (a stopping variable
              finishes at its improve phase); it then does nothing else
  Stopper   = the reference puts a stopping variable back in ok mode after _send_ok (:529), so when no neighbour
              stopped with it, it completes the next ok phase once more (its neighbours' End arrive later)

The per-variable state is what the variable computed in the last phase it completed: a variable that finished by
flood keeps the values of its previous phases (the reference's partial updates from messages that arrived before
its End are not part of the state).  Random draws: Philox4x32-10 with counter (canonical variable id, cycle, 0, 0),
cycle 0xffffffff for the start value of every variable, else the reference's cycle_count (round - 1).
"""
import numpy as np

import philox
from _mgm2_oracle import neighbour_lists, var_constraints

LIVE = 2 ** 31 - 1
ROW_KEYS = ("eval", "improve", "new_value", "can_move", "qlm", "consistent", "counter", "finish_phase",
            "violated", "weight")


class DbaOracle:
    """Lock-step DBA.  State after `init()` == fixture row 0, after n `step()` == row n."""

    def __init__(self, inst, dtype=np.float64, mode="min", infinity=10000, max_distance=50, stop_cycle=0, seed=0,
                 var_id=None, **_ignored):
        if mode != "min":
            raise ValueError("DBA is a constraint **satisfaction** algorithm and only support minimization "
                             "objective")
        self.T = np.float64 if np.dtype(dtype) == np.float64 else np.float32
        self.infinity, self.max_distance = int(infinity), int(max_distance)
        self.stop_cycle, self.seed = int(stop_cycle or 0), int(seed)
        self.dom = [int(x) for x in inst["dom_size"]]
        V = self.V = len(self.dom)
        fp = [int(x) for x in inst["factor_ptr"]]
        ev = [int(x) for x in inst["edge_var"]]
        self.scope = [ev[fp[f]:fp[f + 1]] for f in range(len(fp) - 1)]
        tsize = [int(np.prod([self.dom[u] for u in sc])) for sc in self.scope]
        toff = [0] + list(np.cumsum(tsize, dtype=np.int64))
        if "table_off" in inst and inst["table_off"] is not None:
            toff = [int(x) for x in inst["table_off"]]
        tables = np.ascontiguousarray(inst["tables"], dtype=self.T)
        self.bad = [tables[toff[f]:toff[f] + tsize[f]] >= self.T(self.infinity) for f in range(len(tsize))]
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
        rank = inst["var_rank"] if "var_rank" in inst else None
        self.rank = [int(x) for x in rank] if rank is not None else list(range(V))
        self.var_id = [int(x) for x in var_id] if var_id is not None else list(range(V))
        self.cycle = 0

    # -- pieces of the reference computation --------------------------------------------------
    def violated_at(self, v, k, x, val):
        """rel(x) >= infinity (:478) for slot k of v, the other variables at `val`."""
        f = self.cons[v][k]
        i = 0
        for u, s in zip(self.scope[f], self.strides[f]):
            i += (x if u == v else val[u]) * s
        return bool(self.bad[f][i])

    def evals(self, v, val):
        """compute_eval_value of every value (:452-482) and the violated slots at the current value."""
        ev = [0] * self.dom[v]
        for k in range(len(self.cons[v])):
            w = self.weight[v][k]
            for x in range(self.dom[v]):
                if self.violated_at(v, k, x, val):
                    ev[x] += w
        viol = [self.violated_at(v, k, val[v], val) for k in range(len(self.cons[v]))]
        return ev, viol

    # -- lifecycle -----------------------------------------------------------------------------
    def init(self):
        V = self.V
        self.val = []
        for v in range(V):   # on_start (:341-349): always a draw, initial_value is ignored
            _, w = philox.draw(self.seed, self.var_id[v], philox.INIT_CYCLE)
            self.val.append(philox.choice_index(w, self.dom[v]))
        self.cost = [None] * V
        self.weight = [[1] * len(self.cons[v]) for v in range(V)]
        self.violated = [[False] * len(self.cons[v]) for v in range(V)]
        self.counter_own = [0] * V
        self.eval, self.improve, self.counter = [0] * V, [0] * V, [0] * V
        self.new_value = [-1] * V
        self.can_move, self.qlm, self.consistent = [False] * V, [False] * V, [False] * V
        self.finish = [LIVE] * V
        self.live = sum(1 for v in range(V) if self.nbrs[v])
        self.end_round = LIVE if self.live else 0
        self.rounds = 0          # rounds enqueued
        self.cycle = 0
        self.unresolved = 0
        self.stats = dict(rank_decided=0, multi_draws=0, weight_raises=0, moves=0, stops=0, floods=0,
                          evals_after_stop=0)
        return self

    @property
    def ended(self):
        return self.end_round != LIVE

    @property
    def finished(self):
        """Every variable with neighbours finished, or stop_cycle reached (gdba_gpu's convention)."""
        return self.ended or bool(self.stop_cycle and self.rounds + 1 >= self.stop_cycle)

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.rounds += 1
            if self.end_round >= self.rounds:
                self._round(self.rounds)
            self.cycle = min(self.rounds, self.end_round)
        return self

    def _finish(self, v, p, k):
        self.finish[v] = p
        self.live -= 1
        if self.live == 0:
            self.end_round = k

    def _flooded(self, v, p):
        return any(self.finish[u] < p for u in self.nbrs[v])

    def _round(self, k):
        V, val = self.V, self.val
        conn = [v for v in range(V) if self.nbrs[v]]
        p = 2 * k
        for v in conn:   # ok phase (:366-420)
            # a variable that stopped in the last improve phase is back in ok mode (_go_to_wait_ok_mode runs after
            # _send_ok, :529): it evaluates once more when no neighbour stopped with it
            if self.finish[v] not in (LIVE, p - 1):
                continue
            if self._flooded(v, p):
                if self.finish[v] == LIVE:
                    self._finish(v, p, k)
                    self.stats["floods"] += 1
                continue
            if self.finish[v] != LIVE:
                self.stats["evals_after_stop"] += 1
            ev, viol = self.evals(v, val)
            cur = ev[val[v]]
            best, bests = self.infinity, []
            for x in range(self.dom[v]):
                if ev[x] < best:
                    best, bests = ev[x], [x]
                elif ev[x] == best:
                    bests.append(x)
            g = cur - best
            cons = cur == 0
            cm, nv = g > 0, -1
            if cm:
                if not bests:           # the reference raises on random.choice([]): keep the value
                    self.unresolved += 1
                    cm = False
                else:
                    _, w = philox.draw(self.seed, self.var_id[v], k - 1)
                    nv = bests[philox.choice_index(w, len(bests))]
                    self.stats["multi_draws"] += len(bests) >= 2
            self.eval[v], self.improve[v], self.new_value[v] = cur, g, nv
            self.cost[v] = cur          # the reference assigns its current_cost field directly (:385)
            self.counter[v] = self.counter_own[v] if cons else 0
            self.can_move[v], self.qlm[v], self.consistent[v] = cm, g <= 0, cons
            self.violated[v] = viol
        p = 2 * k + 1
        new_val = list(val)
        for v in conn:   # improve phase (:504-562)
            if self.finish[v] != LIVE:
                continue
            if self._flooded(v, p):
                self._finish(v, p, k)
                self.stats["floods"] += 1
                continue
            mine = self.improve[v]
            cnt, cm, q, cons = self.counter[v], self.can_move[v], self.qlm[v], self.consistent[v]
            for u in self.nbrs[v]:
                cnt = min(cnt, self.counter[u])
                if self.improve[u] > mine:
                    cm = q = False
                elif self.improve[u] == mine and self.rank[u] < self.rank[v]:
                    if cm:
                        self.stats["rank_decided"] += 1
                    cm = False
                if self.eval[u] > 0:
                    cons = False
            stop = False
            if cons:
                cnt += 1
                stop = cnt == self.max_distance
            self.counter_own[v] = cnt
            self.can_move[v], self.qlm[v], self.consistent[v] = cm, q, cons
            if stop:
                self._finish(v, p, k)
                self.stats["stops"] += 1
                continue
            if q:
                for s, bad in enumerate(self.violated[v]):
                    if bad:
                        self.weight[v][s] += 1
                        self.stats["weight_raises"] += 1
            if cm:
                new_val[v] = self.new_value[v]
                self.cost[v] = self.eval[v] - mine
                self.stats["moves"] += 1
        self.val = new_val

    # -- views -----------------------------------------------------------------------------------
    def values(self):
        """(value index per variable, current cost or NaN while the reference's is None)."""
        cost = np.array([np.nan if c is None else float(c) for c in self.cost])
        return np.array(self.val, dtype=np.int32), cost

    def record(self):
        """The per-round fixture arrays (ROW_KEYS) of the current state."""
        b = lambda a: np.array(a, dtype=np.uint8)  # noqa: E731
        return dict(eval=np.array(self.eval, dtype=np.int64), improve=np.array(self.improve, dtype=np.int64),
                    new_value=np.array(self.new_value, dtype=np.int32), can_move=b(self.can_move), qlm=b(self.qlm),
                    consistent=b(self.consistent), counter=np.array(self.counter, dtype=np.int32),
                    finish_phase=np.array(self.finish, dtype=np.int32),
                    violated=b([x for row in self.violated for x in row]),
                    weight=np.array([w for row in self.weight for w in row], dtype=np.int32))
