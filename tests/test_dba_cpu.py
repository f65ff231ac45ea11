"""DBA on the CPU: the oracle (tests/_dba_oracle.py) against the reference's own lock-step trajectories
(tests/golden/dba_*.npz, written by tools/make_golden_dba.py from the unmodified pydcop/algorithms/dba.py), what
those fixtures exercise, and the fixture regeneration where the reference is present."""
import os
import subprocess
import sys
from collections import deque

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _dba_oracle import LIVE, ROW_KEYS, DbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names

DBA_FIXTURES = golden_names("dba_")


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def end_round(inst, k):
    """Round in which the last variable with neighbours finished, by row k (LIVE while one is live)."""
    fp = inst["finish_phase"][k]
    conn = has_neighbours(inst)
    if conn.any() and (fp[conn] == LIVE).any():
        return LIVE
    return int(fp[conn].max()) // 2 if conn.any() else 0


def has_neighbours(inst):
    o = DbaOracle(inst)
    return np.array([bool(n) for n in o.nbrs])


def check_trajectory(run, inst, meta, name, rows=None):
    """Compare `run` (init()/step()/values()/record()/cycle) with a fixture round by round: values, costs and every
    ROW_KEYS array after every round, and the cycle the engine reports."""
    n = meta["n_cycles"] if rows is None else rows
    for k in range(n + 1):
        if k:
            run.step()
        val, cost = run.values()
        assert np.array_equal(val, inst["value"][k]), (name, k, "value")
        assert np.array_equal(cost, inst["cost"][k], equal_nan=True), (name, k, "cost")
        rec = run.record()
        for key in ROW_KEYS:
            assert np.array_equal(rec[key], inst[key][k]), (name, k, key, rec[key], inst[key][k])
        assert run.cycle == min(k, end_round(inst, k)), (name, k, run.cycle)


def oracle_for(inst, meta, dt=np.float64):
    return DbaOracle(inst, dt, seed=meta["seed"], **meta["params"])


@pytest.mark.parametrize("name", DBA_FIXTURES)
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_oracle_reproduces_reference_trajectory(name, dt):
    """Every fixture's entries compare with infinity the same way in f32, so both precisions follow it."""
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, dt).init(), inst, meta, name)


def distances(o, src):
    d = [None] * o.V
    d[src] = 0
    q = deque([src])
    while q:
        v = q.popleft()
        for u in o.nbrs[v]:
            if d[u] is None:
                d[u] = d[v] + 1
                q.append(u)
    return d


def behaviours(name):
    """Which of the behaviours the fixtures are meant to show this fixture shows."""
    inst, meta = load(name)
    o = oracle_for(inst, meta).init().step(meta["n_cycles"])
    conn = has_neighbours(inst)
    fp = inst["finish_phase"][-1]
    inf, tables = meta["params"]["infinity"], inst["tables"]
    out = set()
    if (fp[conn] != LIVE).all():
        out.add("all_finish")
        if len(set(fp[conn])) == 1 and fp[conn][0] % 2 == 1:
            out.add("simultaneous_stop")
    if (fp[conn] == LIVE).all():
        out.add("no_stop")
    if ((fp != LIVE) & (fp % 2 == 0)).any():
        out.add("flood")
    done = fp[fp != LIVE]
    if len(done):
        p0 = int(done.min())
        k = p0 // 2
        dist = distances(o, int(np.nonzero(fp == p0)[0][0]))
        for u in range(o.V):
            if dist[u] == 3 and fp[u] == p0 + 3 and k + 1 <= meta["n_cycles"] \
                    and inst["value"][k + 1][u] != inst["value"][k][u]:
                out.add("post_stop_move_d3")
    if inst["weight"][-1].max() > 1:
        out.add("weights_grow")
    if (tables == inf).any():
        out.add("equal_infinity")
    if ((tables < inf) & (tables > inf - 1)).any():
        out.add("below_infinity")
    if np.isinf(tables).any():
        out.add("inf_entries")
    if o.stats["rank_decided"]:
        out.add("rank_decided")
    if o.stats["multi_draws"]:
        out.add("multi_draws")
    if o.stats["evals_after_stop"]:
        out.add("eval_after_stop")
    iv = inst["init_value"]
    if (iv >= 0).any() and (inst["value"][0][iv >= 0] != iv[iv >= 0]).any():
        out.add("initial_ignored")
    return out


@pytest.mark.parametrize("name", DBA_FIXTURES)
def test_fixture_shows_what_it_is_meant_to(name):
    _, meta = load(name)
    missing = set(meta["shows"]) - behaviours(name)
    assert not missing, (name, missing)


def test_fixture_set_covers_the_quirks():
    names = set(DBA_FIXTURES)
    assert {"dba_ref_gc_csp", "dba_max_distance_0", "dba_max_distance_1", "dba_infinity_100", "dba_rand_d12",
            "dba_k4_unsat", "dba_ring_flood", "dba_initial_values"} <= names
    assert load("dba_rand_d12")[0]["dom_size"].max() == 12
    assert load("dba_infinity_100")[1]["params"]["infinity"] == 100
    assert load("dba_ref_gc_csp")[1]["params"] == {"infinity": 10000, "max_distance": 3, "stop_cycle": 0}
    shapes = dict(iso=0, uno=0, ranks=0)
    for n in DBA_FIXTURES:
        inst, meta = load(n)
        o = oracle_for(inst, meta)
        for v in range(o.V):
            if not o.nbrs[v]:
                shapes["uno" if o.cons[v] else "iso"] += 1
                # never evaluates, moves or finishes: keeps its random start value
                assert (inst["value"][:, v] == inst["value"][0, v]).all() and (inst["finish_phase"][:, v] == LIVE).all()
        shapes["ranks"] += not np.array_equal(inst["var_rank"], np.arange(o.V))
        arities = {len(s) for s in o.scope}
        if n.startswith("dba_mixed"):
            assert arities == {1, 2, 3}
    assert all(shapes.values()), shapes


def test_stop_cycle_and_steps_after_the_end():
    inst, meta = load("dba_coloring_same_round")
    o = DbaOracle(inst, seed=meta["seed"], **dict(meta["params"], stop_cycle=6)).init().step(50)
    assert o.cycle == 5 and o.finished and not o.ended
    assert np.array_equal(o.values()[0], inst["value"][5])
    o = oracle_for(inst, meta).init().step(meta["n_cycles"])
    assert o.finished and o.ended
    c, rec = o.cycle, o.record()
    o.step(5)
    assert o.cycle == c and all(np.array_equal(rec[k], o.record()[k]) for k in ROW_KEYS)


def test_unresolved_keeps_the_value():
    """Weights past infinity: improve > 0 but no value below infinity (the reference raises on
    random.choice([])); the oracle keeps the value and counts the case."""
    from test_mgm2_cpu import unit_instance
    inst = unit_instance([[0, 1], [0, 1]], [([0, 1], lambda a, b: float("inf"))])
    o = DbaOracle(inst, infinity=1, max_distance=0, seed=3).init()
    o.weight = [[5], [5]]
    o.val = [0, 0]
    o.step()
    assert o.unresolved >= 1 and o.val[0] == 0


def test_mode_max_refused():
    inst, meta = load("dba_ref_gc_csp")
    with pytest.raises(ValueError, match="only support minimization"):
        DbaOracle(inst, mode="max")


# ---- regeneration against the live reference ------------------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


@needs_ref
def test_regeneration_reproduces_committed_fixtures(tmp_path):
    names = [n for n in DBA_FIXTURES if n != "dba_ref_gc_csp"] + ["dba_ref_gc_csp"]
    script = ("import sys; sys.path.insert(0, %r)\n" % os.path.join(ROOT, "tools")
              + "import make_golden_dba as m; m.main(%r, %r)\n" % (names, str(tmp_path)))
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    for n in names:
        a, _ = orc.load_golden(os.path.join(GOLDEN_DIR, n + ".npz"))
        b, _ = orc.load_golden(os.path.join(str(tmp_path), n + ".npz"))
        assert set(a) == set(b)
        for k in a:
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), (n, k)
