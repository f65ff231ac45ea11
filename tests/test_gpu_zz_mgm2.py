"""GPU: MGM-2 kernels (pydcop_b200/csrc/mgm2.cu) through the C-ABI against the reference's own
lock-step trajectories (tests/golden/mgm2_*.npz), against the oracle (tests/_mgm2_oracle.py) on
larger random graphs, and one drop-in `pydcop solve --algo mgm2_gpu` run with the real engine."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _mgm2_oracle import Mgm2Oracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200.layout import layout_from_instance
from test_mgm2_cpu import check_trajectory
from test_mgm2_hostshim import _assert_same, random_mgm2_instance

pytestmark = pytest.mark.gpu


def _engine(inst, precision, meta, **kw):
    from pydcop_b200.engine import Mgm2Engine
    return Mgm2Engine(layout_from_instance(inst), precision=precision, mode=meta["mode"], seed=meta["seed"],
                      var_rank=inst["var_rank"], **dict(meta["params"], **kw))


@pytest.mark.parametrize("name", golden_names("mgm2_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_mgm2_matches_fixture(name, precision):
    """f64 (and f32 on integer costs) against the reference's trajectory; f32 on float costs against
    the f32 oracle."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = _engine(inst, precision, meta).init()
    if precision == "f64" or "float" not in name:
        check_trajectory(eng, inst, meta, dt, name)
    else:
        o = Mgm2Oracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
        for k in range(1, meta["n_cycles"] + 1):
            o.step()
            eng.step()
            _assert_same(eng.record(), o.record(), dt, k)
            assert np.array_equal(eng.values()[0], o.values()[0]), k
            assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k
    assert eng.launch_count == 1 + 5 * eng.cycle


@pytest.mark.parametrize("precision,mode,favor,threshold,levels", [("f64", "min", "unilateral", 0.5, 0),
                                                                  ("f32", "max", "no", 0.6, 0),
                                                                  ("f32", "max", "no", 0.5, 2),
                                                                  ("f64", "min", "coordinated", 0.5, 2)])
def test_mgm2_matches_oracle_on_random_graphs(precision, mode, favor, threshold, levels):
    """20k variables, mixed arities 2 / 3 / 1, float tables or integer costs with few levels (ties that
    the favor rule decides): every array of every cycle bit-identical to the oracle in the same
    precision."""
    from pydcop_b200.engine import Mgm2Engine
    inst = random_mgm2_instance(20000, 4 if not levels else 3, [2, 3, 1], seed=7, levels=levels)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, favor=favor, threshold=threshold, seed=19)
    o = Mgm2Oracle(inst, dt, **kw).init()
    eng = Mgm2Engine(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    assert np.array_equal(eng.values()[0], o.values()[0])
    pairs = 0
    for k in range(1, 5):
        o.step()
        eng.step()
        rec = o.record()
        _assert_same(eng.record(), rec, dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k
        pairs += int(rec["go"].sum())
    assert pairs > 100
    if levels:
        assert o.stats["ties"] > 0
        if favor == "no":
            assert o.stats["coin_commit"] > 0 and o.stats["coin_refuse"] > 0
        else:
            assert o.stats["tie_commits"] == o.stats["ties"]


def test_mgm2_stop_cycle_and_chunked_steps():
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "mgm2_default.npz"))
    a = _engine(inst, "f64", meta, stop_cycle=6).init()
    a.step(50)
    assert a.cycle == 5 and a.finished           # rounds run = stop_cycle - 1 (mgm2.py:613)
    assert a.launch_count == 1 + 5 * 5
    b = _engine(inst, "f64", meta).init()
    for _ in range(5):
        b.step()
    va, ca = a.values()
    vb, cb = b.values()
    assert np.array_equal(va, vb) and np.array_equal(ca, cb, equal_nan=True)
    assert np.array_equal(va, inst["value"][5])


def test_mgm2_solution_cost():
    from pydcop_b200 import ingest, solve as S
    path = os.path.join(ROOT, "tests", "golden", "instances", "graph_coloring_10_4_15_0.1.yml")
    res = S.solve(path, "mgm2", {"stop_cycle": 20}, precision="f64", seed=4)
    d = ingest.load_yaml(path)
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    viol, cost = S.solution_cost(d, idx)
    assert res["status"] == "FINISHED" and res["cycle"] == 20 and res["algo"] == "mgm2"
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
    inst = d.instance()
    if inst.get("var_ptr") is None:
        from pydcop_b200.layout import default_var_csr
        inst["var_ptr"], inst["var_edge"] = default_var_csr(d.n_vars, inst["edge_var"])
    inst["var_rank"] = S.name_rank(d)
    o = Mgm2Oracle(inst, np.float64, mode=d.objective, seed=4, stop_cycle=20).init().step(20)
    assert np.array_equal(idx, o.values()[0])


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_mgm2_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo mgm2_gpu and the real engine behind the proxies: the
    run FINISHES at stop_cycle with a full assignment whose cost the reference reports.  One agent hosts every
    computation: the offer-sized communication loads of MGM-2 (the reference's formula) leave `adhoc` no feasible
    distribution of this instance over its agents, for the reference's mgm2 as well."""
    from pydcop_b200 import ingest
    path = os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "mgm2_gpu", "--algo_params", "stop_cycle:25",
                                       "--algo_params", "seed:3", "-d", "oneagent", path])
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=240,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout[r.stdout.index("{"):r.stdout.rindex("}") + 1])
    assert res["status"] == "FINISHED", (res, r.stderr[-1500:])
    assert len(res["assignment"]) == 10 and res["cycle"] >= 24
    from pydcop_b200 import solve as S
    d = ingest.load_yaml(path)
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    viol, cost = S.solution_cost(d, idx)
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
    assert viol <= 3      # 10 variables, 3 colours: a local search leaves at most a few conflicts
