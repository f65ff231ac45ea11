"""GPU: GDBA kernels (pydcop_b200/csrc/gdba.cu) through the C-ABI against the reference's own
lock-step trajectories (tests/golden/gdba_*.npz), against the oracle (tests/_gdba_oracle.py) on
larger random graphs, and one drop-in `pydcop solve --algo gdba_gpu` run with the real engine."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _gdba_oracle import GdbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200.layout import layout_from_instance
from test_gdba_cpu import check_trajectory
from test_gdba_hostshim import MODE_GRID, compare_with_oracle, random_gdba_instance

pytestmark = pytest.mark.gpu


def _engine(inst, precision, meta, **kw):
    from pydcop_b200.engine import GdbaEngine
    return GdbaEngine(layout_from_instance(inst), precision=precision, mode=meta["mode"], seed=meta["seed"],
                      var_rank=inst["var_rank"], **dict(meta["params"], **kw))


@pytest.mark.parametrize("name", golden_names("gdba_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_gdba_matches_fixture(name, precision):
    """f64 (and f32 on integer costs) against the reference's trajectory; f32 on float costs against
    the f32 oracle."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = _engine(inst, precision, meta).init()
    if precision == "f64" or "float" not in name:
        check_trajectory(eng, inst, meta, dt, name)
    else:
        o = GdbaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
        compare_with_oracle(eng, o, dt, meta["n_cycles"])
    assert eng.launch_count == 1 + 2 * eng.cycle


@pytest.mark.parametrize("modifier,increase_mode", MODE_GRID)
def test_gdba_matches_oracle_on_random_graphs(modifier, increase_mode):
    """20k variables, mixed arities 2 / 3 / 1, variable costs: every array of every round bit-identical
    to the oracle in the same precision (f64 float costs in min mode for A, f32 integer costs in max
    mode for M)."""
    from pydcop_b200.engine import GdbaEngine
    if modifier == "A":
        precision, mode, violation, levels = "f64", "min", "NZ", 0
    else:
        precision, mode, violation, levels = "f32", "max", "NM", 3
    inst = random_gdba_instance(20000, 3, seed=17, levels=levels)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, modifier=modifier, violation=violation, increase_mode=increase_mode, seed=23)
    o = GdbaOracle(inst, dt, **kw).init()
    eng = GdbaEngine(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    compare_with_oracle(eng, o, dt, 4)
    assert o.stats["breakouts"] > 100
    if increase_mode != "T":
        assert o.stats["span_increases"] > 0


def test_gdba_stop_cycle_chunked_steps_and_launches():
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "gdba_A_NZ_E.npz"))
    a = _engine(inst, "f64", meta, stop_cycle=6).init()
    a.step(50)
    assert a.cycle == 5 and a.finished           # rounds run = stop_cycle - 1, as mgm_gpu
    assert a.launch_count == 1 + 2 * 5
    b = _engine(inst, "f64", meta).init()
    for _ in range(5):
        b.step()
    va, ca = a.values()
    vb, cb = b.values()
    assert np.array_equal(va, vb) and np.array_equal(ca, cb, equal_nan=True)
    assert np.array_equal(a.modifiers(), b.modifiers())
    assert np.array_equal(va, inst["value"][5]) and np.array_equal(a.modifiers(), inst["modifiers"][5])
    a.init()                                     # init restarts: modifiers back to base
    assert a.cycle == 0 and np.array_equal(a.modifiers(), inst["modifiers"][0])


def test_gdba_solution_cost():
    from pydcop_b200 import ingest, solve as S
    path = os.path.join(ROOT, "tests", "golden", "instances", "graph_coloring_10_4_15_0.1.yml")
    res = S.solve(path, "gdba", {"stop_cycle": 21, "increase_mode": "T"}, precision="f64", seed=4)
    d = ingest.load_yaml(path)
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    viol, cost = S.solution_cost(d, idx)
    assert res["status"] == "FINISHED" and res["cycle"] == 21 and res["algo"] == "gdba"
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
    inst = d.instance()
    if inst.get("var_ptr") is None:
        from pydcop_b200.layout import default_var_csr
        inst["var_ptr"], inst["var_edge"] = default_var_csr(d.n_vars, inst["edge_var"])
    inst["var_rank"] = S.name_rank(d)
    o = GdbaOracle(inst, np.float64, mode=d.objective, seed=4, increase_mode="T", stop_cycle=21).init().step(21)
    assert np.array_equal(idx, o.values()[0])


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_gdba_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo gdba_gpu and the real engine behind the proxies: the
    run FINISHES at stop_cycle with a full assignment whose cost the reference reports.  One agent
    hosts every computation, as for mgm2_gpu."""
    from pydcop_b200 import ingest
    path = os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "gdba_gpu", "--algo_params", "stop_cycle:25",
                                       "--algo_params", "seed:3", "--algo_params", "increase_mode:T",
                                       "-d", "oneagent", path])
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
