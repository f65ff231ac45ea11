"""MGM-2 on the CPU: the oracle (tests/_mgm2_oracle.py) against the reference's own lock-step
trajectories (tests/golden/mgm2_*.npz, written by tools/make_golden_mgm2.py from the unmodified
pydcop/algorithms/mgm2.py), the reference's unit-test answers, the host arrays of the engine, and
the fixture regeneration / a fuzz against the live reference where the reference is present."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _mgm2_oracle import Mgm2Oracle, draw
from conftest import GOLDEN_DIR, ROOT, golden_names

import philox

MGM2_FIXTURES = golden_names("mgm2_")
ROW_KEYS = ("local_cost", "offerer", "partner", "committed", "gain", "potential_value", "go")


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def check_trajectory(run, inst, meta, dt, name):
    """Compare `run` (init()/step()/values()/record()/cycle) with a fixture, row by row; f32 runs
    compare with the fixture rounded to f32 where the fixture is exact in f32."""
    conn = ~np.isnan(inst["gain"][1]) if meta["n_cycles"] else None
    for k in range(meta["n_cycles"] + 1):
        ran = False
        if k:
            before = run.cycle
            run.step()
            ran = run.cycle > before
        val, cost = run.values()
        assert np.array_equal(val, inst["value"][k]), (name, k, "value")
        known = ~np.isnan(inst["cost"][k])
        assert np.array_equal(~np.isnan(cost), known), (name, k)
        assert np.array_equal(cost[known].astype(dt), inst["cost"][k][known].astype(dt)), (name, k, "cost")
        if ran:
            rec = run.record()
            for key in ROW_KEYS:
                got, want = rec[key], inst[key][k]
                if key in ("local_cost", "gain"):
                    assert np.array_equal(got[conn].astype(dt), want[conn].astype(dt)), (name, k, key)
                else:
                    assert np.array_equal(got, want), (name, k, key)
    assert run.cycle + 1 == int(inst["cycle_count"][-1].max()) or not meta["params"]["stop_cycle"]


def oracle_for(inst, meta, dt):
    return Mgm2Oracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"])


def test_fixture_set_is_complete():
    assert len(MGM2_FIXTURES) >= 15
    inst, _ = load("mgm2_mixed_arity")
    assert set(np.diff(inst["factor_ptr"])) == {1, 2, 3}


@pytest.mark.parametrize("name", MGM2_FIXTURES)
def test_oracle_f64_reproduces_reference_trajectory(name):
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, np.float64).init(), inst, meta, np.float64, name)


@pytest.mark.parametrize("name", [n for n in MGM2_FIXTURES if "float" not in n])
def test_oracle_f32_reproduces_integer_cost_fixtures(name):
    """Integer costs are exact in f32: the f32 oracle takes the same decisions."""
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, np.float32).init(), inst, meta, np.float32, name)


def test_fixtures_exercise_every_branch():
    seen = {k: 0 for k in ("offers", "commits", "go", "pair_moves", "refused", "unary_only")}
    for name in MGM2_FIXTURES:
        inst, meta = load(name)
        N = meta["n_cycles"]
        seen["offers"] += int(inst["offerer"][1:].sum())
        seen["commits"] += int((inst["committed"][1:] & (inst["offerer"][1:] == 0)).sum())
        seen["go"] += int(inst["go"][1:].sum())
        seen["refused"] += int((inst["offerer"][1:] & (inst["committed"][1:] == 0)).sum())
        for k in range(1, N + 1):
            moved = inst["value"][k] != inst["value"][k - 1]
            seen["pair_moves"] += int((moved & (inst["committed"][k] == 1)).sum())
    for name in ("mgm2_threshold0",):
        inst, _ = load(name)
        assert inst["offerer"].sum() == 0
    inst, _ = load("mgm2_threshold1")
    conn = ~np.isnan(inst["gain"][1])
    assert inst["committed"].sum() == 0 and (inst["offerer"][1:] == conn).all()
    assert all(v > 0 for k, v in seen.items() if k != "unary_only"), seen


def test_favor_fixtures_exercise_the_favor_rule():
    """The three favor fixtures run the same instance, on which the best offer's global gain equals
    the unilateral gain (the only case `favor` decides) in many cycles.  Their trajectories come from
    the reference; the oracle reproduces them (above) and counts what the rule did."""
    runs = {}
    for favor in ("unilateral", "no", "coordinated"):
        inst, meta = load("mgm2_favor_" + favor)
        assert meta["params"]["favor"] == favor
        o = oracle_for(inst, meta, np.float64).init().step(meta["n_cycles"])
        runs[favor] = (inst, o.stats)
    base, st = runs["unilateral"]
    assert st["ties"] >= 5 and st["tie_commits"] == 0
    st = runs["no"][1]
    assert st["coin_commit"] > 0 and st["coin_refuse"] > 0       # the coin falls on both sides of 0.5
    st = runs["coordinated"][1]
    assert st["tie_commits"] == st["ties"] > 0
    for favor in ("no", "coordinated"):
        inst = runs[favor][0]
        assert np.array_equal(inst["tables"], base["tables"])
        assert not np.array_equal(inst["value"], base["value"]), favor
        assert not np.array_equal(inst["committed"], base["committed"]), favor
    assert not np.array_equal(runs["no"][0]["value"], runs["coordinated"][0]["value"])


def test_stop_cycle_fixture_finishes():
    inst, meta = load("mgm2_stop8")
    assert inst["finished"].all()
    assert int(inst["cycle_count"][-1].max()) == 8
    o = oracle_for(inst, meta, np.float64).init().step(50)
    assert o.cycle == 7 and o.finished


def test_variable_costs_are_ignored():
    """MGM-2's costs use assignment_cost without variable costs: the trajectory of the
    var-costs fixture is the oracle's on the instance with every variable cost zeroed."""
    inst, meta = load("mgm2_var_costs")
    assert np.any(inst["unary"] != 0)
    zero = dict(inst, unary=np.zeros_like(inst["unary"]))
    check_trajectory(oracle_for(zero, meta, np.float64).init(), inst, meta, np.float64, "var_costs")


def test_draw_purpose_zero_is_the_existing_draw():
    for v, c in ((0, 1), (5, philox.INIT_CYCLE), (123, 77)):
        assert draw(99, v, c, 0) == philox.draw(99, v, c)
        assert draw(99, v, c, 1) != philox.draw(99, v, c)


# ---- the reference's unit tests (tests/unit/test_algorithms_mgm2.py), re-asserted on the oracle ----
def unit_instance(doms, constraints, init=None):
    """Instance of variables with domains `doms` (lists of values) and constraints (scope, function of
    the VALUES); every variable lists the constraints it is in, in order."""
    tables, fp, ev = [], [0], []
    for scope, fn in constraints:
        shape = [len(doms[v]) for v in scope]
        tables.append(np.array([fn(*[doms[v][i] for v, i in zip(scope, idx)]) for idx in np.ndindex(*shape)],
                               dtype=float))
        ev.extend(scope)
        fp.append(len(ev))
    var_con = [[f for f, (scope, _) in enumerate(constraints) if v in scope] for v in range(len(doms))]
    var_ptr = np.concatenate([[0], np.cumsum([len(c) for c in var_con])]).astype(np.int32)
    return dict(dom_size=np.array([len(d) for d in doms], np.int32), factor_ptr=np.array(fp, np.int32),
                edge_var=np.array(ev, np.int32), tables=np.concatenate(tables), var_ptr=var_ptr,
                var_con=np.array([f for c in var_con for f in c], np.int32),
                init_value=np.array(init if init is not None else [-1] * len(doms), np.int32))


PHI_UNARY = ([list(range(5))], [([0], lambda x: 1 if x in [0, 2, 3] else 0)])
PHI_BINARY = ([list(range(2)), list(range(2))], [([0, 1], lambda x1, x2: x1 + x2)])
PHI_TERNARY = ([list(range(2)), list(range(2)), [1]], [([0, 1, 2], lambda x1, x2, x3: x1 + x2 + x3)])


@pytest.mark.parametrize("setup,mode,others,bests,best", [
    (PHI_UNARY, "min", {}, [1, 4], 0),                       # test_best_unary
    (PHI_BINARY, "min", {1: 1}, [0], 1),                     # test_binary_func_min
    (PHI_BINARY, "max", {1: 1}, [1], 2),                     # test_binary_func_max
    (PHI_TERNARY, "min", {1: 1, 2: 0}, [0], 2),              # test_3_ary_func_min (x3 = 1: index 0)
    (PHI_TERNARY, "max", {1: 1, 2: 0}, [1], 3),              # test_3_ary_func_max
])
def test_reference_unit_compute_best_value(setup, mode, others, bests, best):
    o = Mgm2Oracle(unit_instance(*setup), mode=mode).init()
    val = [0] * o.V
    for v, x in others.items():
        val[v] = x
    assert o._best_values(0, val) == (bests, best)


@pytest.mark.parametrize("setup,cases", [
    (PHI_UNARY, [([0], 1)]),                                                           # test_unary_function_relation
    (PHI_BINARY, [([0, 0], 0), ([0, 1], 1), ([1, 0], 1), ([1, 1], 2)]),                # test_binary_func
    (PHI_TERNARY, [([0, 0, 0], 1), ([0, 1, 0], 2), ([1, 0, 0], 2), ([1, 1, 0], 3)]),   # test_3_ary_func
])
def test_reference_unit_compute_cost(setup, cases):
    o = Mgm2Oracle(unit_instance(*setup)).init()
    for val, want in cases:
        assert o._cost(o.cons[0], val) == want


@pytest.mark.parametrize("setup,cases", [
    (PHI_UNARY, [([0], 1), ([1], 0)]),                    # test_current_local_cost_unary
    (PHI_BINARY, [([1, 0], 1), ([0, 0], 0)]),             # test_current_local_cost_binary
    (PHI_TERNARY, [([1, 0, 0], 2), ([0, 0, 0], 1)]),      # test_current_local_cost_3_ary
])
def test_reference_unit_current_local_cost(setup, cases):
    """_current_local_cost: the cost of the variable's own value over its constraints; it is the
    local cost the oracle computes in the value phase of x1."""
    inst = unit_instance(*setup)
    for val, want in cases:
        o = Mgm2Oracle(dict(inst, init_value=np.array(val, np.int32))).init()
        assert o._cost(o.cons[0], val) == want
        if o.nbrs[0]:
            o.step()
            assert o.last["local_cost"][0] == want


def test_reference_unit_no_neighbors():
    """test_no_neighbors: max mode, cost x1 * 2 over 0..9: value 9 with cost 18, then finished."""
    o = Mgm2Oracle(unit_instance([list(range(10))], [([0], lambda x1: x1 * 2)]), mode="max").init()
    assert o._best_values(0, [0]) == ([9], 18)
    assert o.val == [9] and o.cost == [18] and o.is_finished == [True]


# ---- regeneration and fuzz against the live reference -------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


def _run_generator(tmp_path, code):
    script = ("import sys; sys.path.insert(0, %r)\n" % os.path.join(ROOT, "tools")) + code
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=str(tmp_path),
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]


@needs_ref
def test_regeneration_reproduces_committed_fixtures(tmp_path):
    names = ["mgm2_ties", "mgm2_mixed_arity", "mgm2_float", "mgm2_favor_no", "mgm2_rand_d12"]
    _run_generator(tmp_path, "import make_golden_mgm2 as m; m.main(%r, %r)\n" % (names, str(tmp_path)))
    for n in names:
        a, _ = orc.load_golden(os.path.join(GOLDEN_DIR, n + ".npz"))
        b, _ = orc.load_golden(os.path.join(str(tmp_path), n + ".npz"))
        assert set(a) == set(b)
        for k in a:
            assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), (n, k)


@needs_ref
def test_fuzz_oracle_against_live_reference(tmp_path):
    """Random instances (mixed arity, float costs, all favor modes, both objectives) through the
    unmodified reference, then through the oracle."""
    code = (
        "import numpy as np, make_golden_mgm2 as m\n"
        "G = m.G\n"
        "for i, (favor, mode, thr) in enumerate([('unilateral', 'min', 0.5), ('no', 'max', 0.3), "
        "('coordinated', 'min', 0.8), ('no', 'min', 0.6)]):\n"
        "    rng = np.random.default_rng(100 + i)\n"
        "    vs, cs = G.random_instance(rng, 22, [4, 3, 2], 34, [2, 3, 2, 1], int_tables=(i % 2 == 0))\n"
        "    vs, cs = m.with_extras(vs, cs)\n"
        "    arr, meta = m.run_mgm2(vs, cs, {'favor': favor, 'threshold': thr}, mode, 10, seed=31 + i)\n"
        "    G.GOLDEN = OUT\n"
        "    G.save('fuzz' + str(i), arr, meta)\n").replace("OUT", repr(str(tmp_path)))
    _run_generator(tmp_path, code)
    for i in range(4):
        inst, meta = orc.load_golden(os.path.join(str(tmp_path), "fuzz%d.npz" % i))
        check_trajectory(oracle_for(inst, meta, np.float64).init(), inst, meta, np.float64, "fuzz%d" % i)
