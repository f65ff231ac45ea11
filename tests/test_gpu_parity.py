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
from _hard_constraints import factor_family
from conftest import GOLDEN_DIR, golden_names

pytestmark = pytest.mark.gpu

# factor / variable kernel selections the environment offers; the hard-constraint fixtures (msx_*, +/-inf
# costs, inf and NaN messages) run under every one of them
KERNEL_CONFIGS = {
    "default": {},
    "pipe": {"PYDCOP_B200_F2V": "pipe", "PYDCOP_B200_V2F": "pipe"},
    "no_tiled_rt": {"PYDCOP_B200_TILED_RT": "0"},
    "no_fast": {"PYDCOP_B200_NO_FAST": "1"},
    "generic_first": {"PYDCOP_B200_FAST_FIRST": "0"},
}
CASES = [pytest.param(n, "default", id=n) for n in golden_names("ms_")] + \
        [pytest.param(n, c, id=f"{n}-{c}") for n in golden_names("msx_") for c in KERNEL_CONFIGS]


def _engine_state(eng):
    q, r = eng.messages()
    fl = eng.flags()
    val, cost = eng.values()
    return q, r, fl, val, cost


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("name,config", CASES)
def test_maxsum_engine_bit_exact_vs_oracle(name, config, precision, monkeypatch):
    """Messages (NaN where the oracle has NaN), send flags, gate counters, values and reported costs at
    every cycle; f64 also against the reference's own trajectory."""
    from pydcop_b200 import MaxSumEngine, layout_from_instance
    for k, v in KERNEL_CONFIGS[config].items():
        monkeypatch.setenv(k, v)
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
        where = (name, config, k)
        assert np.array_equal(q, o.q.astype(np.float64), equal_nan=True), (where, "q")
        assert np.array_equal(r, o.r.astype(np.float64), equal_nan=True), (where, "r")
        assert np.array_equal(fl["q_sent"], o.q_sent), (where, "q_sent")
        assert np.array_equal(fl["r_sent"], o.r_sent), (where, "r_sent")
        assert np.array_equal(fl["r_cnt"] >> 1, o.r_flags >> 2), (where, "r count")
        assert np.array_equal(fl["q_cnt"] >> 1, o.q_flags >> 2), (where, "q count")
        assert np.array_equal(val, o.value), (where, "value")
        assert np.array_equal(cost, o.value_cost.astype(np.float64), equal_nan=True), (where, "value_cost")
        if precision == "f64":  # directly against the reference's trajectory
            assert np.array_equal(q, inst["q_state"][k], equal_nan=True), (where, "q vs reference")
            assert np.array_equal(r, inst["r_state"][k], equal_nan=True), (where, "r vs reference")
            assert np.array_equal(fl["q_sent"].astype(bool), inst["q_sent"][k]), (where, "q_sent vs reference")
            assert np.array_equal(fl["r_sent"].astype(bool), inst["r_sent"][k]), (where, "r_sent vs reference")


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_hard_constraint_fixtures_reach_every_factor_kernel(precision):
    """In the default configuration the msx_* fixtures put factor classes on the warp, the pipelined and
    the runtime-shape kernels, each class on the family tests/_hard_constraints.py expects (the CPU test
    of the fixtures' all-NaN sites relies on that mapping)."""
    from pydcop_b200 import MaxSumEngine, layout_from_instance
    seen = set()
    for name in golden_names("msx_"):
        inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
        L = layout_from_instance(inst)
        plan = MaxSumEngine(L, precision=precision, mode=meta["mode"]).kernel_plan()
        assert plan == [factor_family(tuple(c.dom[:c.arity])) for c in L.classes], (name, plan)
        seen.update(plan)
    assert {"warp", "pipe", "tiled_rt"} <= seen, seen


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
