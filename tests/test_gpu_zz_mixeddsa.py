"""GPU: the MixedDSA kernel (pydcop_b200/csrc/mixeddsa.cu) through the C-ABI against the reference's own lock-step
trajectories (tests/golden/mixeddsa_*.npz), against the oracle (tests/_mixeddsa_oracle.py) on 20k-variable mixed
graphs and at the shape limits, on a second device, through solve(), and one drop-in `pydcop solve --algo
mixeddsa_gpu` run with the real engine."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _mixeddsa_oracle import MixedDsaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200.layout import layout_from_instance
from test_mixeddsa_cpu import EXACT_F32, check_trajectory
from test_mixeddsa_hostshim import LIMITS, compare_with_oracle, limits_instance, random_mixed
from test_mixeddsa_plugin_cpu import HARD_YAML

pytestmark = pytest.mark.gpu


def _engine(inst, precision, meta, **kw):
    from pydcop_b200.engine import MixedDsaEngine
    return MixedDsaEngine(layout_from_instance(inst), precision=precision, mode=meta["mode"], seed=meta["seed"],
                          **dict(meta["params"], **kw))


@pytest.mark.parametrize("name", golden_names("mixeddsa_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_mixeddsa_matches_fixture(name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = _engine(inst, precision, meta).init()
    if precision == "f64" or name in EXACT_F32:
        check_trajectory(eng, inst, meta, dt, name)
    else:
        o = MixedDsaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
        compare_with_oracle(eng, o, dt, meta["n_cycles"])
    n_classes = len(eng.layout.classes)
    assert eng.launch_count == n_classes + 1 + eng.cycle


def test_step_chunks_equal_single_steps_and_stop_cycle():
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "mixeddsa_proba_1.npz"))
    a = _engine(inst, "f64", meta, stop_cycle=9).init()
    a.step(50)
    assert a.cycle == 9 and a.finished          # dsa_gpu's convention: stop_cycle rounds
    b = _engine(inst, "f64", meta).init()
    for _ in range(9):
        b.step()
    va, ca = a.values()
    vb, cb = b.values()
    assert np.array_equal(va, vb) and np.array_equal(ca, cb, equal_nan=True)
    assert np.array_equal(va, inst["value"][9])
    a.init()
    assert a.cycle == 0 and np.array_equal(a.values()[0], inst["value"][0])


@pytest.mark.parametrize("precision,mode,variant,neg", [("f64", "min", "B", False), ("f32", "max", "A", False),
                                                        ("f32", "min", "C", True)])
def test_mixeddsa_matches_oracle_on_random_graphs(precision, mode, variant, neg):
    """20k variables, arities 1-4, hard and soft constraints, dyadic variable costs, initial values."""
    inst = random_mixed(20000, seed=31, levels=4, neg=neg)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, variant=variant, proba_hard=0.8, proba_soft=0.6, seed=13)
    o = MixedDsaOracle(inst, dt, **kw).init()
    from pydcop_b200.engine import MixedDsaEngine
    eng = MixedDsaEngine(layout_from_instance(inst), precision=precision, **kw).init()
    compare_with_oracle(eng, o, dt, 3)


@pytest.mark.parametrize("case", list(LIMITS))
def test_mixeddsa_at_the_limits(case):
    from pydcop_b200.engine import MixedDsaEngine
    inst = limits_instance(case)
    kw = dict(mode="min", variant="B", proba_hard=0.9, proba_soft=0.9, seed=23)
    for precision, dt in (("f64", np.float64), ("f32", np.float32)):
        o = MixedDsaOracle(inst, dt, **kw).init()
        eng = MixedDsaEngine(layout_from_instance(inst), precision=precision, **kw).init()
        compare_with_oracle(eng, o, dt, 3)


def test_mixeddsa_on_a_second_device():
    """A handle on cuda:1 while cuda:0 is current: every launch runs on the handle's device."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from pydcop_b200.engine import MixedDsaEngine
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "mixeddsa_defaults.npz"))
    torch.cuda.set_device(0)
    eng = MixedDsaEngine(layout_from_instance(inst), device="cuda:1", precision="f64", mode=meta["mode"],
                         seed=meta["seed"], **meta["params"]).init()
    check_trajectory(eng, inst, meta, np.float64, "mixeddsa_defaults")
    assert eng.value[0].device.index == 1 and torch.cuda.current_device() == 0


def test_mixeddsa_solve_reports_solution_cost(tmp_path):
    from pydcop_b200 import ingest, solve as S
    from pydcop_b200.layout import default_var_csr
    path = tmp_path / "hard.yaml"
    path.write_text(HARD_YAML)
    res = S.solve(str(path), "mixeddsa", {"stop_cycle": 50}, precision="f64", seed=4)
    d = ingest.load_yaml(str(path))
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    viol, cost = S.solution_cost(d, idx)
    assert res["status"] == "FINISHED" and res["cycle"] == 50 and res["algo"] == "mixeddsa"
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
    inst = d.instance()
    if inst.get("var_ptr") is None:
        inst["var_ptr"], inst["var_edge"] = default_var_csr(d.n_vars, inst["edge_var"])
    o = MixedDsaOracle(inst, np.float64, mode=d.objective, seed=4, stop_cycle=50).init().step(50)
    assert np.array_equal(idx, o.values()[0])


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_mixeddsa_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo mixeddsa_gpu and the real engine behind the proxies: the run
    FINISHES at stop_cycle with the oracle's assignment for the same seed."""
    from pydcop_b200 import ingest
    from pydcop_b200.layout import default_var_csr
    path = tmp_path / "hard.yaml"
    path.write_text(HARD_YAML)
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "mixeddsa_gpu", "--algo_params", "stop_cycle:30",
                                       "--algo_params", "seed:3", "-d", "oneagent", str(path)])
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=240,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout[r.stdout.index("{"):r.stdout.rindex("}") + 1])
    assert res["status"] == "FINISHED", (res, r.stderr[-1500:])
    assert {"assignment", "cost", "violation", "cycle"} <= set(res)
    d = ingest.load_yaml(str(path))
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    inst = d.instance()
    if inst.get("var_ptr") is None:
        inst["var_ptr"], inst["var_edge"] = default_var_csr(d.n_vars, inst["edge_var"])
    o = MixedDsaOracle(inst, np.float64, mode=d.objective, seed=3, stop_cycle=30).init().step(30)
    assert np.array_equal(idx, o.values()[0])
