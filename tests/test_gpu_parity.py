"""GPU parity (run on an H100): CUDA engine through the C-ABI vs the CPU oracle and vs the
reference's own lock-step trajectories (tests/golden, made from the unmodified reference).

Bar (north_star): integer assignments bit-exact; float messages within 1e-5 relative.  What is
actually asserted is stronger: the engine is BIT-IDENTICAL to the same-precision oracle at every
cycle (messages, send decisions, values, reported costs), in f64 and f32; and the f64 engine is
bit-identical to the Python reference's messages.
"""
import os

import numpy as np
import pytest

import oracle as orc
from conftest import GOLDEN_DIR, golden_names

pytestmark = pytest.mark.gpu


def _engine_state(eng):
    q, r = eng.messages()
    fl = eng.flags()
    val, cost = eng.values()
    return q, r, fl, val, cost


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("name", golden_names("ms_"))
def test_maxsum_engine_bit_exact_vs_oracle(name, precision):
    from pydcop_b200 import MaxSumEngine, layout_from_instance
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    npdt = np.float64 if precision == "f64" else np.float32
    o = orc.MaxSumOracle(inst, npdt, mode=meta["mode"], **meta["params"]).init()
    p = {k: v for k, v in meta["params"].items() if k != "noise"}
    eng = MaxSumEngine(layout_from_instance(inst), precision=precision, mode=meta["mode"], **p).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            o.step()
            eng.step()
        q, r, fl, val, cost = _engine_state(eng)
        assert np.array_equal(q, o.q.astype(np.float64)), (name, k, "q")
        assert np.array_equal(r, o.r.astype(np.float64)), (name, k, "r")
        assert np.array_equal(fl["q_sent"], o.q_sent), (name, k, "q_sent")
        assert np.array_equal(fl["r_sent"], o.r_sent), (name, k, "r_sent")
        assert np.array_equal(val, o.value), (name, k, "value")
        assert np.array_equal(cost, o.value_cost.astype(np.float64)), (name, k, "value_cost")
        if precision == "f64":  # directly against the reference's trajectory
            assert np.array_equal(q, inst["q_state"][k]), (name, k, "q vs reference")
            assert np.array_equal(r, inst["r_state"][k]), (name, k, "r vs reference")
            assert np.array_equal(fl["q_sent"].astype(bool), inst["q_sent"][k]), (name, k)
            assert np.array_equal(fl["r_sent"].astype(bool), inst["r_sent"][k]), (name, k)


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("name", golden_names("dsa_"))
def test_dsa_engine_exact_vs_reference(name, precision):
    from pydcop_b200 import DsaEngine, layout_from_instance
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    eng = DsaEngine(layout_from_instance(inst), precision=precision, mode=meta["mode"],
                    seed=meta["seed"], **meta["params"]).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            eng.step()
        assert np.array_equal(eng.values(), inst["value"][k]), (name, k)
    assert eng.cycle == int(inst["cycle_count"][-1].max())


def test_multi_cycle_step_equals_single_steps():
    from pydcop_b200 import MaxSumEngine, layout_from_instance
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, "ms_rand_bin_d10.npz"))
    a = MaxSumEngine(layout_from_instance(inst), precision="f32").init().step(12)
    b = MaxSumEngine(layout_from_instance(inst), precision="f32").init()
    for _ in range(12):
        b.step()
    for x, y in zip(a.messages(), b.messages()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.values()[0], b.values()[0])
    assert a.launch_count == b.launch_count > 0


@pytest.mark.parametrize("name", ["ms_rand_mixed", "ms_arity4_mixed", "ms_gc10_default"])
def test_solution_cost_kernel(name):
    """fg_solution_cost (dcop.py:319-367) against a numpy evaluation of the same assignment."""
    from pydcop_b200 import MaxSumEngine, layout_from_instance
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    p = {k: v for k, v in meta["params"].items() if k != "noise"}
    eng = MaxSumEngine(layout_from_instance(inst), precision="f64", mode=meta["mode"], **p).init().step(15)
    val, _ = eng.values()
    cost, viol = eng.solution_cost(infinity=1e300, unary=inst["unary"])
    expect = 0.0
    fp, ev, toff = inst["factor_ptr"], inst["edge_var"], inst["table_off"]
    for f in range(len(fp) - 1):
        scope = ev[fp[f]:fp[f + 1]]
        shape = tuple(int(inst["dom_size"][v]) for v in scope)
        t = np.asarray(inst["tables"][toff[f]:toff[f + 1]]).reshape(shape)
        expect += float(t[tuple(int(val[v]) for v in scope)])
    uoff = np.concatenate([[0], np.cumsum(inst["dom_size"])])
    expect += float(sum(inst["unary"][uoff[v] + val[v]] for v in range(len(val))))
    assert viol == 0
    assert abs(cost - expect) <= 1e-9 * max(1.0, abs(expect))
