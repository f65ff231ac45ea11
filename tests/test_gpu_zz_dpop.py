"""GPU: DPOP kernels (pydcop_b200/csrc/dpop.cu) through the C-ABI against the reference's own messages
(tests/golden/dpop_*.npz) and against the oracle (tests/_dpop_oracle.py) on a deep and a wide instance."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from _dpop_oracle import DpopOracle
import ref_shim
from conftest import ROOT
from pydcop_b200 import pseudotree as pt
from pydcop_b200.layout import build_layout
from test_dpop_cpu import NAMES, _integer_without_sentinel, check_against_golden, load, same, tree_of

pytestmark = pytest.mark.gpu


def _engine(inst, tree, precision, mode):
    from pydcop_b200.engine import DpopEngine
    L = build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"],
                     unary=inst.get("unary") if hasattr(inst, "get") else inst["unary"])
    return DpopEngine(L, tree, precision=precision, mode=mode).init().step()


def _check_engine(eng, tree, util_ref, value, cost, dt):
    arena = eng.arena.double().cpu().numpy()
    for u in range(tree.n_vars):
        if tree.parent[u] >= 0:
            off = eng._util_off[u]
            tab = arena[off:off + tree.util_size[u]]
            assert same(tab, np.asarray(util_ref(u), dtype=dt).astype(np.float64).reshape(-1)), u
    v, c = eng.values()
    assert np.array_equal(v, value)
    assert same(c, np.asarray(cost, dtype=dt).astype(np.float64))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_dpop_matches_fixture(name, precision):
    """f64 against the reference's UTIL messages, values and costs; f32 too on integer fixtures without
    sentinels, else against the f32 oracle."""
    inst, meta = load(name)
    dt = np.float64 if precision == "f64" else np.float32
    t = tree_of(inst)
    eng = _engine(inst, t, precision, meta["mode"])
    assert eng.finished and eng.launch_count == eng.sched.n_launches
    if precision == "f64" or _integer_without_sentinel(inst):
        check_against_golden(inst, meta, t, lambda u: eng.util(u)[1], *eng.values(), dt)
    o = DpopOracle(inst, t, dt, meta["mode"]).run()
    _check_engine(eng, t, lambda u: o.util[u], o.value, o.cost, dt)
    assert eng.unresolved == o.unresolved
    assert (eng.unresolved > 0) == (meta["error"] == "IndexError")


def test_dpop_deep_instance_matches_oracle():
    """10^5 variables, d = 10, small separators: the light-path kernel over a deep DFS tree."""
    from pydcop_b200.generators import bounded_separator_instance
    inst = bounded_separator_instance(100_000, 10, back=1, span=3, p_back=0.2, seed=3, float_costs=True)
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    eng = _engine(inst, t, "f64", "min")
    s = eng.sched
    assert t.height > 10_000 and s.rounds <= int(np.log2(t.n_vars)) + 1
    assert eng.launch_count == s.n_launches
    o = DpopOracle(inst, t, np.float64, "min").run()
    _check_engine(eng, t, lambda u: o.util[u], o.value, o.cost, np.float64)


def test_dpop_wide_instance_matches_oracle_and_solution_cost():
    """Separators of 6 at d = 10 (joined tables of 10^7 entries) on the grid-wide kernel, with light nodes
    above and below a big one; the roots' costs are the assignment's cost."""
    from pydcop_b200.generators import bounded_separator_instance
    inst = bounded_separator_instance(40, 10, back=5, span=1, seed=4)
    # one pendant variable on every fifth chain variable: light leaves hanging below big nodes
    hosts = np.arange(0, 40, 5)
    inst["dom_size"] = np.concatenate([inst["dom_size"], np.full(len(hosts), 10, dtype=np.int32)])
    inst["edge_var"] = np.concatenate([inst["edge_var"], np.stack([hosts, 40 + np.arange(len(hosts))], 1).reshape(-1)]).astype(np.int32)
    inst["factor_ptr"] = np.arange(0, len(inst["edge_var"]) + 1, 2)
    inst["tables"] = np.concatenate([inst["tables"], np.random.default_rng(5).integers(0, 10, len(hosts) * 100)])
    inst["unary"] = np.zeros(int(inst["dom_size"].sum()))
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    eng = _engine(inst, t, "f32", "max")
    s = eng.sched
    assert max(t.util_size[u] * 10 for u in s.big_nodes) >= 10 ** 7
    big = set(s.big_nodes)
    light = [u for u in range(t.n_vars) if u not in big]

    def ancestors(u):
        while t.parent[u] >= 0:
            u = int(t.parent[u])
            yield u
    assert any(a in big for u in light for a in ancestors(u))          # a light node below a big one
    assert any(a in light for u in big for a in ancestors(u))          # and one above
    assert eng.launch_count == s.n_launches
    o = DpopOracle(inst, t, np.float32, "max").run()
    _check_engine(eng, t, lambda u: o.util[u], o.value, o.cost, np.float32)
    cost, viol = eng.solution_cost()
    assert viol == 0 and cost == pytest.approx(sum(o.cost[r] for r in t.roots), rel=1e-5)


def test_dpop_arena_larger_than_the_device_raises_before_allocating():
    """A clique of 8 variables at d = 256: the deepest separator has 7 variables, 256^7 entries."""
    import torch
    from pydcop_b200._cabi import EngineError
    n, d = 8, 256
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
    inst = dict(dom_size=np.full(n, d, dtype=np.int32), factor_ptr=np.arange(0, 2 * len(pairs) + 1, 2),
                edge_var=np.array(pairs, dtype=np.int32).reshape(-1), tables=np.zeros(len(pairs) * d * d),
                unary=np.zeros(n * d))
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    before = torch.cuda.memory_allocated()
    with pytest.raises(EngineError, match="largest separator") as e:
        _engine(inst, t, "f64", "min")
    assert f"needs {sum(t.util_size) * 8} bytes" in str(e.value)
    assert f"{len(max(t.sep, key=len))} variables" in str(e.value)
    assert torch.cuda.memory_allocated() == before


def test_dpop_solve_entry():
    from pydcop_b200 import ingest, solve as S
    path = os.path.join(ROOT, "tests", "golden", "instances", "graph_coloring_10_4_15_0.1.yml")
    res = S.solve(path, "dpop", precision="f64")
    assert res["status"] == "FINISHED" and res["algo"] == "dpop" and res["cycle"] == 0
    d = ingest.load_yaml(path)
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    viol, cost = S.solution_cost(d, idx)
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
    inst, meta = load("dpop_ref_gc_10_4_15_0_1")
    assert np.array_equal(idx, inst["value"])
    with pytest.raises(ValueError):
        S.solve(path, "dpop", {"stop_cycle": 3})


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_dpop_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo dpop_gpu and the real engine behind the proxies: FINISHED at
    cycle 0 with the reference's optimal assignment (tests/golden/dpop_ref_gc_10_4_15_0_1.npz)."""
    path = os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "dpop_gpu", "-d", "oneagent", path])
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=240,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout[r.stdout.index("{"):r.stdout.rindex("}") + 1])
    assert res["status"] == "FINISHED" and res["cycle"] == 0, (res, r.stderr[-1500:])
    from pydcop_b200 import ingest, solve as S
    d = ingest.load_yaml(path)
    idx = np.array([d.values_of(i).index(res["assignment"][n]) for i, n in enumerate(d.var_names)])
    inst, _ = load("dpop_ref_gc_10_4_15_0_1")
    assert np.array_equal(idx, inst["value"])
    viol, cost = S.solution_cost(d, idx)
    assert res["violation"] == viol and res["cost"] == pytest.approx(cost)
