"""GPU: the factor side's 8-bit table copy (csrc/table_i8.cuh, maxsum_warp.cuh k_f2v_warp with TT = int8_t).

Integer tables in [-128, 127] are read by the warp factor kernel as signed bytes; the decode is exact, so messages,
send decisions, counters and values stay bit-identical to the CPU oracle.  Every compiled warp domain size, both
precisions and both modes, with factor counts that leave a partial last tile; one entry out of the rule (128, 0.5,
-0.0, NaN, inf) keeps the class at full width; a two-shard run on one device takes the 8-bit path too."""
import numpy as np
import pytest

import oracle as orc
from bench import oracle_instance
from pydcop_b200.generators import random_factor_graph

pytestmark = pytest.mark.gpu

WARP_DOMS = [4, 6, 8, 10, 16, 20]


def _int8_instance(d, seed, n_factors=None):
    n_vars = 900 if d <= 10 else 400
    n_factors = n_factors or (16 * (n_vars // 8) + 7)   # not a multiple of the 16-factor tile
    inst = random_factor_graph(n_vars, d, n_factors, 2, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    t = rng.integers(-128, 128, size=len(inst["tables"])).astype(np.float32)
    t[:2] = (-128, 127)
    inst["tables"] = t
    return inst


def _check(eng, o, tag):
    q, r = eng.messages()
    val, cost = eng.values()
    fl = eng.flags()
    assert np.array_equal(q, o.q.astype(np.float64)), (tag, "q")
    assert np.array_equal(r, o.r.astype(np.float64)), (tag, "r")
    assert np.array_equal(val, o.value), (tag, "value")
    assert np.array_equal(cost, o.value_cost.astype(np.float64)), (tag, "value_cost")
    assert np.array_equal(fl["q_sent"], o.q_sent) and np.array_equal(fl["r_sent"], o.r_sent), (tag, "sent")
    assert np.array_equal(fl["q_cnt"] >> 1, o.q_flags >> 2) and np.array_equal(fl["r_cnt"] >> 1, o.r_flags >> 2), (tag, "cnt")


def _run(inst, precision, cycles=6, **params):
    from pydcop_b200 import MaxSumEngine, build_layout
    L = build_layout(**inst)
    dt = np.float64 if precision == "f64" else np.float32
    eng = MaxSumEngine(L, precision=precision, **params).init()
    o = orc.MaxSumOracle(oracle_instance(inst, L), dt, **params).init()
    for k in range(cycles):
        if k:
            eng.step()
            o.step()
        _check(eng, o, (precision, params, k))
    return L, eng


def _widths(L, eng):
    """table width of every binary warp class"""
    return {w for c, w, fam in zip(L.classes, eng.table_widths(), eng.kernel_plan()) if fam == "warp"}


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("d", WARP_DOMS)
def test_int8_tables_equal_oracle(d, precision, mode):
    inst = _int8_instance(d, seed=60 + d)
    L, eng = _run(inst, precision, mode=mode)
    assert _widths(L, eng) == {1}


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("d", [6, 10])
def test_int8_tables_no_damping(d, precision):
    inst = _int8_instance(d, seed=80 + d)
    L, eng = _run(inst, precision, cycles=8, damping_nodes="none")
    assert _widths(L, eng) == {1}


@pytest.mark.parametrize("bad", [128.0, 0.5, -0.0, float("nan"), float("inf")])
@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_one_entry_out_of_rule_keeps_full_width(bad, precision):
    inst = _int8_instance(10, seed=5)
    inst["tables"][777] = bad
    L, eng = _run(inst, precision)
    assert _widths(L, eng) == {4 if precision == "f32" else 8}


def test_float_tables_stay_full_width():
    from pydcop_b200 import MaxSumEngine, build_layout
    inst = random_factor_graph(500, 10, 1000, 2, seed=3, int_tables=False)
    L = build_layout(**inst)
    eng = MaxSumEngine(L, precision="f32")
    assert _widths(L, eng) == {4}


def test_two_shards_on_int8_path_equal_single_gpu():
    from pydcop_b200 import MaxSumEngine, build_layout
    from test_gpu_sharded import _run_sharded
    inst = _int8_instance(10, seed=11, n_factors=3007)
    cycles = 9
    L = build_layout(**inst)
    ref = MaxSumEngine(L, precision="f32").init().step(cycles)
    assert _widths(L, ref) == {1}
    ref_q, ref_r = ref.messages()
    ref_val = ref.values()[0]
    shards = _run_sharded(inst, 2, cycles)
    dom = inst["dom_size"][inst["edge_var"]]
    off = np.concatenate([[0], np.cumsum(dom)])
    val = np.full(len(inst["dom_size"]), -1)
    for s in shards:
        Ls = s.plan.layout
        assert 1 in set(w for c, w in zip(Ls.classes, s.engine.table_widths()) if c.arity == 2 and c.n_factors)
        ids, v = s.local_values()
        val[ids] = v
        q, r = s.engine.messages()
        loff = np.concatenate([[0], np.cumsum(Ls.canon_dom_size[Ls.canon_edge_var])])
        canon = np.concatenate([s.plan.own_factor_edges, s.plan.stub_edges])
        for le, ge in enumerate(canon):
            d = int(dom[ge])
            assert np.array_equal(r[loff[le]:loff[le] + d], ref_r[off[ge]:off[ge] + d]), ("r", ge)
            assert np.array_equal(q[loff[le]:loff[le] + d], ref_q[off[ge]:off[ge] + d]), ("q", ge)
    assert np.array_equal(val, ref_val)
