"""GPU: the SyncBB kernel (pydcop_b200/csrc/syncbb.cu) through the C-ABI against the reference's own message traces
(tests/golden/syncbb_*.npz) and the oracle (tests/_syncbb_oracle.py): every fixture in both precisions, a random
instance of about 10^5 messages, runs split into launches of 1, 7 and everything, the shape limits (domains of 256,
a chain whose path does not fit in shared memory, a hub), solve()'s timeout, and an engine on a second device."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle as orc
from _syncbb_oracle import SyncbbOracle
import ref_shim
from conftest import GOLDEN_DIR, ROOT
from pydcop_b200.layout import layout_from_instance
from test_syncbb_cpu import RUNNABLE
from test_syncbb_hostshim import random_instance, same_message

pytestmark = pytest.mark.gpu


def _engine(inst, precision, mode, device=None):
    from pydcop_b200.engine import SyncbbEngine
    return SyncbbEngine(layout_from_instance(inst), device=device, precision=precision, mode=mode,
                        var_rank=inst.get("var_rank"))


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def same_state(eng, o):
    assert np.array_equal(eng.values(), o.values())
    assert np.array_equal(eng.bounds(), o.bounds())
    assert (eng.steps, eng.messages, eng.finished) == (o.steps, o.messages, o.finished)
    assert np.array_equal(eng.cycle_counts(), o.cycle_counts()) and eng.cycle == int(o.cycle_counts().max())
    kind, recv, plen, ub, fin = eng.message()
    assert same_message((kind, recv, plen, ub), o.message())


@pytest.mark.parametrize("name", RUNNABLE)
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_fixture_matches_oracle(name, precision):
    inst, meta = load(name)
    dt = np.float64 if precision == "f64" else np.float32
    eng = _engine(inst, precision, meta["mode"]).init().step(10 ** 9)
    o = SyncbbOracle(inst, dt, meta["mode"], inst["var_rank"]).init().run()
    same_state(eng, o)
    assert eng.finished and eng.messages == int(inst["msg_count"]) and eng.steps == int(inst["n_steps"])
    if precision == "f64":
        assert np.array_equal(eng.values(), inst["final_sel"])


@pytest.mark.parametrize("name", ["syncbb_tuto", "syncbb_floats", "syncbb_inf"])
def test_one_step_launches_follow_the_trace(name):
    """1-step launches: after every message the same bounds and selections as the reference's trace (f64)."""
    inst, meta = load(name)
    eng = _engine(inst, "f64", meta["mode"]).init()
    n = min(int(inst["n_steps"]), 400)
    for k in range(n):
        kind, recv, plen, _, _ = eng.message()
        assert (kind, recv, plen) == (inst["step_type"][k], inst["step_recv"][k], inst["step_plen"][k]), k
        eng.step(1)
        assert np.array_equal(eng.bounds(), inst["ub"][k]) and np.array_equal(eng.values(), inst["sel"][k]), k


def big_random():
    """About 1.4 * 10^5 messages: 22 variables, shuffled names, float costs with some inf entries."""
    return random_instance(22, 3, 34, seed=4, mode_inf=0.02)


@pytest.mark.parametrize("split", [1, 7, None])
def test_resume_gives_the_same_state(split):
    """A run split into launches of 1, 7 or all messages ends in the oracle's state (the state lives in global
    memory between launches)."""
    inst = big_random()
    o = SyncbbOracle(inst, np.float64, "min", inst["var_rank"]).init().run()
    assert 5 * 10 ** 4 <= o.steps <= 10 ** 6, o.steps
    eng = _engine(inst, "f64", "min").init()
    if split is None:
        eng.step(10 ** 9)
    else:
        for _ in range((o.steps + split - 1) // split):
            eng.step(split)
    same_state(eng, o)


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_large_random_instance(precision):
    dt = np.float64 if precision == "f64" else np.float32
    inst = big_random()
    o = SyncbbOracle(inst, dt, "min", inst["var_rank"]).init().run()
    eng = _engine(inst, precision, "min").init().step(10 ** 9)
    same_state(eng, o)


def test_domain_256():
    """256 candidates per step: the whole block, both selections (first accepted, first strict best)."""
    rng = np.random.default_rng(3)
    inst = dict(dom_size=np.array([256, 256, 5], np.int32), factor_ptr=np.array([0, 2, 4]),
                edge_var=np.array([0, 1, 1, 2], np.int32),
                tables=np.concatenate([rng.integers(0, 50, 256 * 256), rng.integers(0, 50, 256 * 5)]).astype(float))
    for precision, dt in (("f64", np.float64), ("f32", np.float32)):
        for mode in ("min", "max"):
            o = SyncbbOracle(inst, dt, mode).init().run(20000)
            eng = _engine(inst, precision, mode).init().step(o.steps)
            same_state(eng, o)


def chain_with_hub(n):
    """A chain x1 - x2 - ... plus a hub x0 joined to every variable and LAST in name order (var_rank), so each of
    its candidates sums n - 1 earlier-neighbour elements; value 0 costs nothing everywhere, so the search walks the
    chain about three times."""
    rng = np.random.default_rng(n)
    pairs = [(i, i + 1) for i in range(1, n - 1)] + [(0, i) for i in range(1, n)]
    tabs = []
    for _ in pairs:
        t = rng.integers(1, 9, size=4).astype(float)
        t[0] = 0.0
        tabs.append(t)
    return dict(dom_size=np.full(n, 2, np.int32), factor_ptr=np.arange(0, 2 * len(pairs) + 1, 2),
                edge_var=np.array(pairs, np.int32).reshape(-1), tables=np.concatenate(tabs),
                var_rank=np.concatenate([[n - 1], np.arange(n - 1)]).astype(np.int32))


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_long_chain_and_hub(precision):
    """3500 variables: the path (12 B per variable in f64) does not fit in the shared-memory copy, in f32 (8 B) it
    does; the hub, last in the chain, has 3499 earlier-neighbour rows to sum per candidate."""
    dt = np.float64 if precision == "f64" else np.float32
    inst = chain_with_hub(3500)
    o = SyncbbOracle(inst, dt, "min", inst["var_rank"]).init().run()
    hub = o.pos[0]
    assert hub == 3499 and len(o.ass[hub]) == 3499
    eng = _engine(inst, precision, "min").init()
    for _ in range(3):
        eng.step((o.steps + 2) // 3)
    same_state(eng, o)
    assert (o.values() == 0).all()


def test_solve_timeout_and_result():
    from pydcop_b200 import solve as S
    from test_syncbb_solve_cpu import fixture_dict
    d, inst = fixture_dict("syncbb_tuto")
    res = S.solve(d, "syncbb", precision="f64")
    assert res["status"] == "FINISHED" and res["cost"] == 12 and res["msg_count"] == 23 and res["cycle"] == 9
    d, inst = fixture_dict("syncbb_name_order")
    res = S.solve(d, "syncbb_gpu", timeout=0.0)
    assert res["status"] == "TIMEOUT" and res["msg_count"] == 1
    d, inst = fixture_dict("syncbb_infeasible")
    res = S.solve(d, "syncbb")
    assert res["assignment"] == {} and res["cost"] is None


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices (cuda:0 and cuda:1)")
def test_second_device():
    inst, meta = load("syncbb_floats")
    o = SyncbbOracle(inst, np.float64, meta["mode"], inst["var_rank"]).init().run()
    with torch.cuda.device(0):
        eng = _engine(inst, "f64", meta["mode"], device="cuda:1").init().step(10 ** 9)
        same_state(eng, o)
        assert torch.cuda.current_device() == 0 and eng.dev["ub"].device == torch.device("cuda:1")


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_pydcop_solve_syncbb_gpu_real_engine(tmp_path):
    """The unmodified reference CLI with --algo syncbb_gpu and the real engine behind the proxies: the reference's
    assignment on graph_coloring_tuto.yaml (all G, cost 12) and its cycle (tests/golden/syncbb_tuto.npz)."""
    path = os.path.join(ref_shim.INSTANCES, "graph_coloring_tuto.yaml")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import ref_shim; ref_shim.install()\n"
            "from pydcop_b200 import launcher\n"
            "launcher.main(%r)\n") % (ROOT, os.path.join(ROOT, "oracle"),
                                      ["-t", "60", "solve", "--algo", "syncbb_gpu", "-d", "oneagent", path])
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=240,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout[r.stdout.index("{"):r.stdout.rindex("}") + 1])
    inst, _ = load("syncbb_tuto")
    assert res["status"] == "FINISHED" and res["cycle"] == int(inst["cycle_count"].max()), (res, r.stderr[-1500:])
    assert res["assignment"] == {"v1": "G", "v2": "G", "v3": "G", "v4": "G"} and res["cost"] == 12
