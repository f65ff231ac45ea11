"""GPU: DBA kernels (pydcop_b200/csrc/dba.cu) through the C-ABI against the reference's own lock-step trajectories
(tests/golden/dba_*.npz), against the oracle (tests/_dba_oracle.py) on larger graphs and at the C-ABI's shape limits,
the early finish of `solve()`, and one drop-in `pydcop solve --algo dba_gpu` run with the real engine."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import _limits as LM
import oracle as orc
import ref_shim
from _dba_oracle import ROW_KEYS, DbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200.layout import layout_from_instance
from test_dba_cpu import check_trajectory, end_round
from test_dba_hostshim import expected_bits, random_dba_instance

pytestmark = pytest.mark.gpu


def _engine(inst, precision, seed, params, **kw):
    from pydcop_b200.engine import DbaEngine
    return DbaEngine(layout_from_instance(inst), precision=precision, seed=seed, var_rank=inst.get("var_rank"),
                     **dict(params, **kw))


def check_bits(eng, precision, infinity):
    dt = np.float64 if precision == "f64" else np.float32
    got = eng.bits[:int(eng.bit_row_bytes // 4)].cpu().numpy().view(np.uint32)
    assert np.array_equal(got, expected_bits(eng.layout, infinity, dt))


def compare_with_oracle(eng, o, n_cycles):
    """Every array of every round bit-identical to the oracle, the same cycle and finish."""
    assert np.array_equal(eng.values()[0], o.values()[0])
    for k in range(1, n_cycles + 1):
        o.step()
        eng.step()
        got, want = eng.record(), o.record()
        for key in ROW_KEYS:
            assert np.array_equal(got[key], want[key]), (k, key)
        v, c = eng.values()
        assert np.array_equal(v, o.values()[0]) and np.array_equal(c, o.values()[1], equal_nan=True), k
        assert eng.cycle == o.cycle and eng.finished == o.finished, k
    assert eng.unresolved == o.unresolved


def init_launches(eng):
    return 1 + (eng.layout.n_edges > 0)


@pytest.mark.parametrize("name", golden_names("dba_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_dba_matches_fixture(name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    eng = _engine(inst, precision, meta["seed"], meta["params"]).init()
    check_bits(eng, precision, meta["params"]["infinity"])
    check_trajectory(eng, inst, meta, name)
    # a round is two launches; none once the end has been observed
    assert eng.launch_count == init_launches(eng) + 2 * eng.cycle
    assert eng.record()["bit_row_bytes"] == eng.bit_row_bytes and eng.unresolved == 0


@pytest.mark.parametrize("precision,max_distance,infinity", [("f64", 2, 10000), ("f32", 3, 100)])
def test_dba_matches_oracle_on_20k_variables(precision, max_distance, infinity):
    """20k variables, arities 2 / 3 / 1, entries at, above and just below infinity: every array of every round
    bit-identical to the oracle, through the first stops, the End flood and the rounds after it."""
    inst = random_dba_instance(20000, 3, seed=17, infinity=infinity)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(infinity=infinity, max_distance=max_distance, seed=23)
    o = DbaOracle(inst, dt, **kw).init()
    eng = _engine(inst, precision, 23, dict(infinity=infinity, max_distance=max_distance)).init()
    check_bits(eng, precision, infinity)
    compare_with_oracle(eng, o, 14)
    assert o.stats["stops"] > 100 and o.stats["floods"] > 100 and o.stats["weight_raises"] > 100


def limit_instance(case):
    inst = (LM.LOCAL[case]() if case in LM.LOCAL
            else LM.with_local_search_arrays(LM.MAXSUM[case](), 7))
    rng = np.random.default_rng(5)
    t = np.asarray(inst["tables"], dtype=np.float64)
    inst["tables"] = np.where(rng.random(len(t)) < 0.4, 10000.0, t)
    return inst


@pytest.mark.parametrize("case", list(LM.LOCAL) + ["arity8_d3", "hub2400", "unary_only", "no_factors"])
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_dba_at_the_limits(case, precision):
    """Domains 1 and 256 (8 words per row), {1, 2, 256}, arity 8, a hub of degree 2400, unary-only and factor-free
    graphs (tests/_limits.py), 40 % of the entries raised to infinity."""
    inst = limit_instance(case)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(max_distance=3, seed=29)
    o = DbaOracle(inst, dt, **kw).init()
    eng = _engine(inst, precision, 29, dict(max_distance=3)).init()
    if eng.layout.n_edges:
        check_bits(eng, precision, 10000)
    compare_with_oracle(eng, o, 5)
    if case in ("unary_only", "no_factors"):   # no variable has a neighbour: finished from the start, cycle 0
        assert eng.finished and eng.cycle == 0 and eng.launch_count == init_launches(eng)


def test_steps_after_the_device_side_finish():
    """Rounds enqueued after every variable finished (before the host looked) change nothing and report the same
    cycle; once observed, steps launch nothing."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "dba_coloring_same_round.npz"))
    eng = _engine(inst, "f64", meta["seed"], meta["params"]).init()
    eng.step(meta["n_cycles"] + 7)      # one call: the end is not observed in between
    n = meta["n_cycles"]
    assert eng.launch_count == init_launches(eng) + 2 * (n + 7)
    assert eng.finished and eng.cycle == end_round(inst, n) < n
    v, c = eng.values()
    assert np.array_equal(v, inst["value"][n]) and np.array_equal(c, inst["cost"][n], equal_nan=True)
    rec = eng.record()
    for key in ROW_KEYS:
        assert np.array_equal(rec[key], inst[key][n]), key
    launches = eng.launch_count
    eng.step(10)
    assert eng.launch_count == launches and eng.cycle == end_round(inst, n)
    eng.init()                           # init restarts
    assert eng.cycle == 0 and not eng.finished and np.array_equal(eng.values()[0], inst["value"][0])


def test_dba_solve_finishes_early():
    from pydcop_b200 import solve as S
    path = os.path.join(ROOT, "tests", "golden", "instances", "graph_coloring_csp.yaml")
    res = S.solve(path, "dba", {"max_distance": 3, "stop_cycle": 100}, precision="f64", seed=4)
    assert res["status"] == "FINISHED" and 0 < res["cycle"] < 99 and res["algo"] == "dba"
    assert res["cost"] == 0 and res["violation"] == 0
    r = subprocess.run([sys.executable, "-m", "pydcop_b200.solve", "-a", "dba", "-p", "max_distance:3", "-p",
                        "stop_cycle:100", path], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout)
    assert out["status"] == "FINISHED" and out["cycle"] < 100 and out["cost"] == 0


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_dba_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo dba_gpu and the real engine behind the proxies: every variable has a
    neighbour, so the run FINISHES when the End flood has reached them all, with a consistent colouring."""
    path = os.path.join(ROOT, "tests", "golden", "instances", "graph_coloring_csp.yaml")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "dba_gpu", "--algo_params", "max_distance:3",
                                       "--algo_params", "seed:3", "-d", "oneagent", path])
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=240,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout[r.stdout.index("{"):r.stdout.rindex("}") + 1])
    assert res["status"] == "FINISHED", (res, r.stderr[-1500:])
    a = res["assignment"]
    assert len(a) == 3 and a["v1"] != a["v2"] and a["v2"] != a["v3"] and res["violation"] == 0


def test_dba_unresolved_keeps_the_value():
    """Weights grown past infinity on the device: the value is kept, nothing is drawn, can_move is cleared and
    every such variable is counted in every round, as the oracle does."""
    from test_dba_hostshim import unresolved_instance
    inst = unresolved_instance()
    kw = dict(infinity=3, max_distance=0)
    o = DbaOracle(inst, seed=2, **kw).init()
    eng = _engine(inst, "f64", 2, kw).init()
    o.weight = [[5] * len(c) for c in o.cons]
    eng.weight.fill_(5)
    start = o.values()[0].copy()
    compare_with_oracle(eng, o, 3)
    rec = eng.record()
    assert eng.unresolved == o.unresolved == 9
    assert (rec["improve"] > 0).all() and (rec["can_move"] == 0).all() and (rec["new_value"] == -1).all()
    assert np.array_equal(eng.values()[0], start)
