"""GDBA on the CPU: the oracle (tests/_gdba_oracle.py) against the reference's own lock-step
trajectories (tests/golden/gdba_*.npz, written by tools/make_golden_gdba.py from the unmodified
pydcop/algorithms/gdba.py), what those fixtures exercise, the reference's unit-test answers, and
the fixture regeneration where the reference is present."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _gdba_oracle import GdbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names

GDBA_FIXTURES = golden_names("gdba_")
ROW_KEYS = ("improve", "new_value", "violated", "breakout", "modifiers")


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def check_trajectory(run, inst, meta, dt, name, rows=None):
    """Compare `run` (init()/step()/values()/record()/modifiers()) with a fixture, round by round;
    f32 runs compare with the fixture rounded to f32."""
    n = meta["n_cycles"] if rows is None else rows
    assert np.array_equal(run.modifiers(), inst["modifiers"][0]), (name, 0, "modifiers")
    for k in range(n + 1):
        if k:
            run.step()
        val, cost = run.values()
        assert np.array_equal(val, inst["value"][k]), (name, k, "value")
        known = ~np.isnan(inst["cost"][k])
        assert np.array_equal(~np.isnan(cost), known), (name, k)
        assert np.array_equal(cost[known].astype(dt), inst["cost"][k][known].astype(dt)), (name, k, "cost")
        if k:
            rec = run.record()
            for key in ROW_KEYS:
                got, want = rec[key], inst[key][k]
                if key == "improve":
                    assert np.array_equal(got.astype(dt), want.astype(dt), equal_nan=True), (name, k, key)
                else:
                    assert np.array_equal(got, want), (name, k, key)


def oracle_for(inst, meta, dt):
    return GdbaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"])


def test_fixture_set_is_complete():
    assert len(GDBA_FIXTURES) == 24 + 7
    grid = {tuple(load(n)[1]["params"][k] for k in ("modifier", "violation", "increase_mode"))
            for n in GDBA_FIXTURES if n.count("_") == 3 and not n.startswith("gdba_max")}
    assert len(grid) == 24
    assert {load(n)[1]["mode"] for n in GDBA_FIXTURES if n.startswith("gdba_max")} == {"max"}
    inst, _ = load("gdba_rand_d12")
    assert inst["dom_size"].max() == 12


@pytest.mark.parametrize("name", GDBA_FIXTURES)
def test_oracle_f64_reproduces_reference_trajectory(name):
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, np.float64).init(), inst, meta, np.float64, name)


@pytest.mark.parametrize("name", [n for n in GDBA_FIXTURES if "float" not in n])
def test_oracle_f32_reproduces_integer_cost_fixtures(name):
    """Integer and dyadic costs are exact in f32: the f32 oracle takes the same decisions."""
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, np.float32).init(), inst, meta, np.float32, name)


def test_fixtures_have_the_required_shapes():
    """Every instance has degree-1 variables, a ternary constraint spanning a variable's
    neighbourhood, a variable without constraints and one with only unary constraints."""
    for name in GDBA_FIXTURES:
        inst, meta = load(name)
        o = oracle_for(inst, meta, np.float64)
        deg = [len(n) for n in o.nbrs]
        assert 1 in deg, name
        assert any(len(o.scope[f]) == 3 and o.span[v][k] for v in range(o.V) for k, f in enumerate(o.cons[v])), name
        assert any(not o.cons[v] for v in range(o.V)), name
        assert any(o.cons[v] and not o.nbrs[v] for v in range(o.V)), name


def test_fixtures_exercise_the_breakout_rules():
    total = dict(rank_decided=0, multi_draws=0)
    for name in GDBA_FIXTURES:
        inst, meta = load(name)
        assert inst["breakout"][1:].sum() > 0, name                 # every fixture breaks out
        o = oracle_for(inst, meta, np.float64).init().step(meta["n_cycles"])
        st = o.stats
        for k in total:
            total[k] += st[k]
        if meta["params"]["increase_mode"] != "T":
            # increases land on spanning constraints; breakouts elsewhere leave the modifiers at base
            assert st["span_increases"] > 0 and st["other_breakout_slots"] > 0, (name, st)
            base = 0 if meta["params"]["modifier"] == "A" else 1
            off = np.concatenate([[0], np.cumsum([o.tsize[f] for v in range(o.V) for f in o.cons[v]])])
            slot = 0
            for v in range(o.V):
                for k in range(len(o.cons[v])):
                    if not o.span[v][k]:
                        assert (inst["modifiers"][-1][off[slot]:off[slot + 1]] == base).all(), (name, v, k)
                    slot += 1
            assert (inst["modifiers"][-1] != base).any(), name
        if meta["mode"] == "max":
            assert st["max_breakouts_next_to_improving"] > 0, (name, st)
    assert total["rank_decided"] > 0 and total["multi_draws"] > 0, total


def test_variable_costs_enter_every_evaluation():
    """The prefix variable-cost term: zeroing the variable costs changes the trajectory."""
    inst, meta = load("gdba_var_costs")
    assert np.any(inst["unary"] != 0)
    zero = dict(inst, unary=np.zeros_like(inst["unary"]))
    a = oracle_for(inst, meta, np.float64).init().step(meta["n_cycles"])
    b = oracle_for(zero, meta, np.float64).init().step(meta["n_cycles"])
    assert a.values()[1].tolist() != b.values()[1].tolist()


def test_stop_cycle():
    inst, meta = load("gdba_A_NZ_E")
    o = GdbaOracle(inst, mode=meta["mode"], seed=meta["seed"], **dict(meta["params"], stop_cycle=6)).init().step(50)
    assert o.cycle == 5 and o.finished
    assert np.array_equal(o.values()[0], inst["value"][5])


# ---- the reference's unit tests (tests/unit/test_algorithms_gdba.py), re-asserted on the oracle ----
def unit(doms, constraints, **kw):
    from test_mgm2_cpu import unit_instance
    o = GdbaOracle(unit_instance(doms, constraints), **kw).init()
    return o


EQ = lambda a, b: 1 if a == b else 0  # noqa: E731
PHI3 = lambda x1, x2, x3: 2 if x1 == x2 else (1 if x1 == x3 else 0)  # noqa: E731


@pytest.mark.parametrize("doms,fn,others,want", [
    ([range(2)] * 2, EQ, {1: 0}, [1, 0]),                                                  # test_compute_eval_binary
    ([range(3)] * 3, lambda a, b, c: 1 if a == b or a == c else 0, {1: 0, 2: 1}, [1, 1, 0]),  # test_compute_eval_3_ary
])
def test_reference_unit_compute_eval(doms, fn, others, want):
    o = unit([list(d) for d in doms], [(list(range(len(doms))), fn)])
    val = [0] * o.V
    for v, x in others.items():
        val[v] = x
    assert [o.eval_value(0, x, val) for x in range(o.dom[0])] == want


@pytest.mark.parametrize("doms,fn,mode,others,bests,best", [
    ([range(2)] * 2, EQ, "min", {1: 0}, [1], 0),                     # test_min_compute_best_for_binary_constraint
    ([range(2)] * 2, EQ, "max", {1: 1}, [1], 1),                     # test_max_compute_best_for_binary_constraint
    ([range(3)] * 3, lambda a, b, c: 1 if a == b or a == c else 0, "min", {1: 0, 2: 0}, [1, 2], 0),
])
def test_reference_unit_best_improvement(doms, fn, mode, others, bests, best):
    o = unit([list(d) for d in doms], [(list(range(len(doms))), fn)], mode=mode)
    val = [0] * o.V
    for v, x in others.items():
        val[v] = x
    assert o.best_values(0, val) == (bests, best)


@pytest.mark.parametrize("modifier,doms,fn,others,entries,want", [
    ("A", [range(3)], lambda x: x, {}, [(0,)], [5, 1, 2]),                                  # test_eff_cost_A_unary
    ("A", [range(3)] * 3, PHI3, {1: 1, 2: 2}, [(0, 1, 2)], [5, 2, 1]),                      # test_eff_cost_A_n_ary
    ("M", [range(3)], lambda x: x, {}, [(0,)], [0, 1, 2]),                                  # test_eff_cost_M_unary
    ("M", [range(3)] * 3, PHI3, {1: 1, 2: 2}, [(0, 1, 2), (1, 1, 2)], [0, 10, 1]),          # test_eff_cost_M_n_ary
])
def test_reference_unit_eff_cost(modifier, doms, fn, others, entries, want):
    """The reference sets modifiers to 5 directly; the only constraint spans x1's neighbourhood."""
    n = len(doms)
    o = unit([list(d) for d in doms], [(list(range(n)), fn)], modifier=modifier)
    o.tab[0][0] = np.zeros(o.tsize[0], dtype=np.int64)
    for e in entries:
        o.tab[0][0][o._index(0, list(e))] = 5 - o.base_mod
    val = [0] * n
    for v, x in others.items():
        val[v] = x
    got = []
    for x in range(3):
        val[0] = x
        got.append(o.eff_cost(0, 0, val))
    assert got == want


@pytest.mark.parametrize("violation,want", [("NZ", [True, True, False]), ("NM", [True, True, False]),
                                            ("MX", [False, True, False])])
def test_violation_modes(violation, want):
    """_is_violated on the base table of PHI3 (entries 0, 1, 2) with x2 = 1, x3 = 0: x1 = 0, 1, 2 gives
    1, 2, 0.  (The reference's TestsConstraintViolation cases are not collected: no test_ prefix.)"""
    o = unit([[0, 1, 2]] * 3, [([0, 1, 2], PHI3)], violation=violation)
    assert [o.is_violated(0, 0, [x, 1, 0]) for x in range(3)] == want


@pytest.mark.parametrize("mode,doms,want", [
    ("E", [range(2)] * 3, {(0, 1, 1): 1}),                                   # test_increase_E
    ("R", [range(2)] * 3, {(0, 1, 1): 1, (1, 1, 1): 1}),                     # test_increase_R
    ("C", [range(3)] * 3, {(0, y, z): 1 for y in range(3) for z in range(3)}),  # test_increase_C
    ("T", [range(2)] * 3, {e: 1 for e in np.ndindex(2, 2, 2)}),             # test_increase_T
])
def test_reference_unit_increase(mode, doms, want):
    o = unit([list(d) for d in doms], [([0, 1, 2], PHI3)], increase_mode=mode)
    o.increase_cost(0, 0, [0, 1, 1])
    for e in np.ndindex(*[len(d) for d in doms]):
        assert o.modifier_at(0, 0, o._index(0, list(e))) == want.get(tuple(e), 0), (mode, e)


def test_increase_on_a_constraint_that_does_not_span():
    """Two binary constraints: E / R / C on one of them change no effective cost, T raises all."""
    doms = [[0, 1]] * 3
    cons = [([0, 1], EQ), ([0, 2], lambda a, b: 1)]
    for mode, want in (("E", 1.0), ("R", 1.0), ("C", 1.0), ("T", 2.0)):
        o = unit(doms, cons, increase_mode=mode)
        o.increase_cost(0, 1, [0, 0, 0])
        for x in range(2):
            for z in range(2):
                assert o.eff_cost(0, 1, [x, 0, z]) == want, mode


# ---- regeneration against the live reference ------------------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


@needs_ref
def test_regeneration_reproduces_committed_fixtures(tmp_path):
    # not gdba_gc10: the YAML loader's variable order follows string hashing, which changes between processes
    names = ["gdba_A_NZ_E", "gdba_M_NM_R", "gdba_max_A_NZ_E", "gdba_float", "gdba_var_costs"]
    script = ("import sys; sys.path.insert(0, %r)\n" % os.path.join(ROOT, "tools")
              + "import make_golden_gdba as m; m.main(%r, %r)\n" % (names, str(tmp_path)))
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    for n in names:
        a, _ = orc.load_golden(os.path.join(GOLDEN_DIR, n + ".npz"))
        b, _ = orc.load_golden(os.path.join(str(tmp_path), n + ".npz"))
        assert set(a) == set(b)
        for k in a:
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), (n, k)
