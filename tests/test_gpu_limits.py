"""GPU: every device engine at the shape limits of the C-ABI (tests/_limits.py): domain sizes 1 and 256
(FG_MAX_DOM), arity 8 (FG_MAX_ARITY), hubs of degree > 2 000, unary-only and factor-free graphs, separators of
32 and 33 variables (FG_DPOP_MAX_SEP).  Each test compares with the same-precision oracle bit for bit at every
cycle, and asserts which kernel family the shape reached, so a change in kernel selection cannot move a shape
off the path it checks."""
import math
import types

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _dpop_oracle import DpopOracle
from _gdba_oracle import GdbaOracle
from _hard_constraints import FAST_DOMS
from _mgm2_oracle import Mgm2Oracle
from bench import oracle_instance
from pydcop_b200 import pseudotree as pt
from pydcop_b200.layout import build_layout, layout_from_instance
from test_gdba_hostshim import compare_with_oracle
from test_gpu_zz_dpop import _check_engine, _engine as _dpop_engine
from test_mgm2_hostshim import _assert_same

pytestmark = pytest.mark.gpu

PRECISIONS = ["f32", "f64"]


def _dt(precision):
    return np.float64 if precision == "f64" else np.float32


# ---------------------------------------------------------------------------------------------------------------
# MaxSum
def _compare_maxsum(eng, o, k):
    q, r = eng.messages()
    val, cost = eng.values()
    fl = eng.flags()
    assert np.array_equal(q, o.q.astype(np.float64), equal_nan=True), ("q", k)
    assert np.array_equal(r, o.r.astype(np.float64), equal_nan=True), ("r", k)
    assert np.array_equal(val, o.value), ("value", k)
    assert np.array_equal(cost, o.value_cost.astype(np.float64), equal_nan=True), ("value_cost", k)
    assert np.array_equal(fl["q_sent"], o.q_sent) and np.array_equal(fl["r_sent"], o.r_sent), ("sent", k)
    assert np.array_equal(fl["r_cnt"] >> 1, o.r_flags >> 2), ("r count", k)
    assert np.array_equal(fl["q_cnt"] >> 1, o.q_flags >> 2), ("q count", k)


MAXSUM_PARAMS = [dict(), dict(mode="max", start_messages="all", damping_nodes="vars")]


@pytest.mark.parametrize("params", MAXSUM_PARAMS, ids=["default", "max_all_vars"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", [c for c in LM.MAXSUM if c != "no_factors"])
def test_maxsum_at_the_limits(case, precision, params):
    from pydcop_b200 import MaxSumEngine
    inst = LM.MAXSUM[case]()
    L = build_layout(**inst)
    dt = _dt(precision)
    o = orc.MaxSumOracle(oracle_instance(inst, L), dt, **params).init()
    eng = MaxSumEngine(L, precision=precision, **params).init()
    fam = eng.kernel_plan()
    assert "generic" not in fam, fam
    elem = np.dtype(dt).itemsize
    for c, f in zip(L.classes, fam):
        shape = c.dom[:c.arity]
        if c.arity >= 4 or len(set(shape)) > 1 or any(x not in FAST_DOMS for x in shape):
            assert f == "tiled_rt", (shape, fam)
    if case in ("d256", "doms_1_3_256"):   # a 256 x 256 table does not fit the kernel's 72 KB: read in place
        assert any(f == "tiled_rt" and c.table_size * elem > 72 * 1024 for c, f in zip(L.classes, fam))
    if case.startswith("arity8"):
        assert any(c.arity == 8 and f == "tiled_rt" for c, f in zip(L.classes, fam))
    if case.startswith("hub"):               # degree > 32: the variable side runs k_v2f_generic for the hub
        deg = np.diff(np.asarray(L.var_ptr))
        assert deg.max() >= 2000 and ((deg >= 17) & (deg <= 32)).sum() >= 2000
    if case == "unary_only":
        assert all(c.arity == 1 for c in L.classes)
    for k in range(9):
        if k:
            o.step()
            eng.step()
        _compare_maxsum(eng, o, k)


@pytest.mark.parametrize("params", MAXSUM_PARAMS, ids=["default", "max_all_vars"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_maxsum_without_factors_steps_as_a_no_op(precision, params):
    """No factor and no edge: the variable side and the two-stream fork are skipped; step(n) changes nothing."""
    from pydcop_b200 import MaxSumEngine
    inst = LM.MAXSUM["no_factors"]()
    L = build_layout(**inst)
    assert L.n_edges == 0 and not L.classes
    o = orc.MaxSumOracle(oracle_instance(inst, L), _dt(precision), **params).init()
    eng = MaxSumEngine(L, precision=precision, **params).init()
    assert eng.kernel_plan() == []
    before = [np.copy(a) for a in (*eng.messages(), *eng.values())]
    _compare_maxsum(eng, o, 0)
    eng.step(5)
    o.step(5)
    _compare_maxsum(eng, o, 5)
    for a, b in zip(before, (*eng.messages(), *eng.values())):
        assert np.array_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# DSA and A-DSA: the generic kernel (k_dsa_step_generic)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case,variant,mode,var_costs", LM.DSA_RUNS)
def test_dsa_generic_kernel_at_the_limits(case, variant, mode, var_costs, precision):
    from pydcop_b200 import DsaEngine
    inst = LM.DSA[case]()
    L = build_layout(**inst)
    dt = _dt(precision)
    kw = dict(mode=mode, variant=variant, seed=7, probability=0.7, var_costs=var_costs)
    o = orc.DsaOracle(oracle_instance(inst, L), dt, **kw).init()
    eng = DsaEngine(L, precision=precision, **kw).init()
    assert eng.tables_or is None and eng.row_cache is None      # neither binary fast path: the generic kernel
    if case == "arity8_d2":
        assert max(c.arity for c in L.classes) == 8
    if case == "hub2400":
        assert np.diff(np.asarray(L.var_ptr)).max() >= 2000
    assert np.array_equal(eng.values(), o.val)
    moved = set()
    for k in range(1, 11):
        prev = o.val.copy()
        o.step()
        eng.step()
        assert np.array_equal(eng.values(), o.val), k
        moved.update(o.val[prev != o.val].tolist())
    if case == "d256_all_tie" and variant == "C":   # every value ties: drop_cur draws among 255
        assert len(moved) > 20 and max(moved) > 200, sorted(moved)


# ---------------------------------------------------------------------------------------------------------------
# MGM
def _run_mgm(inst, precision, mode, cycles=8):
    from pydcop_b200.engine import MgmEngine
    dt = _dt(precision)
    o = orc.MgmOracle(inst, dt, mode=mode, seed=17).init()
    eng = MgmEngine(layout_from_instance(inst), precision=precision, mode=mode, seed=17,
                    var_rank=inst["var_rank"]).init()
    assert np.array_equal(eng.values()[0], o.val)
    moved = 0
    for k in range(1, cycles + 1):
        prev = o.val.copy()
        o.step()
        eng.step()
        val, cost = eng.values()
        assert np.array_equal(val, o.val), k
        assert np.array_equal(cost.astype(dt), o.cost, equal_nan=True), k
        gain, new_value = eng.gains()
        assert np.array_equal(gain.astype(dt), o.gain) and np.array_equal(new_value, o.new_val), k
        moved += int((prev != o.val).sum())
    return eng, moved


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", list(LM.MGM))
def test_mgm_generic_gain_kernel_at_the_limits(case, precision, mode):
    eng, _ = _run_mgm(LM.MGM[case](), precision, mode)
    assert eng.fast_chunk == 0            # k_mgm_gain, the per-thread rel[FG_MAX_DOM] kernel


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("d", [4, 8, 10, 16, 20])
def test_mgm_active_row_kernel_with_a_hub_over_three_chunks(d, precision):
    inst = LM.mgm_hub(d)
    eng, moved = _run_mgm(inst, precision, "max" if d % 8 else "min")
    assert eng.fast_chunk in (2, 4) and eng.row_cache is not None      # k_mgm_gain_cached
    elem = np.dtype(_dt(precision)).itemsize
    spt = 8 if d * elem <= 32 else (4 if d * elem <= 80 else 2)        # csrc/mgm_cached_kernels.cuh MgmCachedCfg
    deg = np.diff(inst["var_ptr"])
    assert deg.max() >= 3 * 128 * spt and (deg == 0).sum() >= 40 and moved > 0


# ---------------------------------------------------------------------------------------------------------------
# MGM-2 and GDBA (their only kernels are the generic ones: rel[FG_MAX_DOM], and MGM-2's cc[FG_MAX_DOM])
@pytest.mark.parametrize("precision,mode,favor", [("f32", "min", "no"), ("f64", "max", "coordinated"),
                                                  ("f32", "max", "unilateral"), ("f64", "min", "no")])
@pytest.mark.parametrize("case", list(LM.LOCAL))
def test_mgm2_at_the_limits(case, precision, mode, favor):
    from pydcop_b200.engine import Mgm2Engine
    inst = LM.LOCAL[case]()
    dt = _dt(precision)
    kw = dict(mode=mode, favor=favor, threshold=0.5, seed=19)
    o = Mgm2Oracle(inst, dt, **kw).init()
    eng = Mgm2Engine(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    assert int(eng.layout.dom_size.max()) == (1 if case == "d1" else 256)
    assert np.array_equal(eng.values()[0], o.values()[0])
    offers = pairs = 0
    for k in range(1, 5):
        o.step()
        eng.step()
        rec = o.record()
        _assert_same(eng.record(), rec, dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k
        offers += int(rec["offerer"].sum())
        pairs += int(rec["go"].sum())
    assert offers > 0
    if case != "d1" and favor != "unilateral":   # one value: nothing to gain; unilateral at d = 256: no pair in 4 cycles
        assert pairs > 0


@pytest.mark.parametrize("precision,mode", [("f64", "min"), ("f32", "max")])
@pytest.mark.parametrize("modifier,increase_mode", LM.GDBA_MODES)
@pytest.mark.parametrize("case", list(LM.LOCAL))
def test_gdba_at_the_limits(case, modifier, increase_mode, precision, mode):
    from pydcop_b200.engine import GdbaEngine
    inst = LM.gdba_instance(case)
    dt = _dt(precision)
    kw = dict(mode=mode, modifier=modifier, violation="NZ", increase_mode=increase_mode, seed=23)
    o = GdbaOracle(inst, dt, **kw).init()
    eng = GdbaEngine(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    assert int(eng.layout.dom_size.max()) == (1 if case == "d1" else 256)
    compare_with_oracle(eng, o, dt, 6)
    if mode == "min":                      # every entry >= 1 violates NZ: minimising meets quasi-local minima
        assert o.stats["breakouts"] > 0
        if increase_mode != "T" and case != "d256":
            assert o.stats["span_increases"] > 0


# ---------------------------------------------------------------------------------------------------------------
# DPOP
def _dpop_against_oracle(inst, precision, mode):
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    eng = _dpop_engine(inst, t, precision, mode)
    assert eng.finished and eng.launch_count == eng.sched.n_launches
    dt = _dt(precision)
    o = DpopOracle(inst, t, dt, mode).run()
    _check_engine(eng, t, lambda u: o.util[u], o.value, o.cost, dt)
    assert eng.unresolved == o.unresolved == 0
    return eng, t


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_dpop_d256_big_nodes_and_value_walk(precision, mode):
    """UTIL tables of 256^2 entries on the grid-wide kernel, VALUE walks with 8 values per lane, ties."""
    inst = LM.dpop_d256()
    eng, t = _dpop_against_oracle(inst, precision, mode)
    assert eng.sched.big_nodes and max(t.util_size[u] for u in eng.sched.big_nodes) == 256 ** 2
    val, _ = eng.values()
    cost, viol = eng.solution_cost()
    terms, _ = LM.cost_terms(inst, val)
    assert viol == 0 and abs(cost - math.fsum(terms)) <= (len(terms) - 1) * 2.0 ** -53 * np.abs(terms).sum()


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_dpop_with_domain_one_variables(precision, mode):
    inst = LM.dpop_with_domain_one()
    eng, t = _dpop_against_oracle(inst, precision, mode)
    assert (inst["dom_size"] == 1).sum() > 20 and not eng.sched.big_nodes      # light-path kernel only


@pytest.mark.parametrize("precision", PRECISIONS)
def test_dpop_separator_of_32_variables(precision):
    inst = LM.clique(33)
    eng, t = _dpop_against_oracle(inst, precision, "min")
    assert max(len(s) for s in t.sep) == pt.MAX_SEP == 32


def test_dpop_separator_of_33_variables_is_refused_before_allocating():
    import ctypes as C
    import torch
    from pydcop_b200 import _cabi, engine as E
    from pydcop_b200._cabi import EngineError
    inst = LM.clique(34)
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    assert max(len(s) for s in t.sep) == 33
    before = torch.cuda.memory_allocated()
    with pytest.raises(EngineError, match="separator of 33 variables: the kernels decode at most 32"):
        _dpop_engine(inst, t, "f64", "min")
    assert torch.cuda.memory_allocated() == before
    # the C-ABI refuses the same descriptor on its own
    L = build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"], unary=inst["unary"])
    inputs, state, scalars = E.dpop_plan(L, t, pt.schedule(t), "f64")
    assert scalars["max_sep"] == 33
    d = _cabi.FgDpopDesc()
    d.abi_version, d.precision = _cabi.FG_ABI_VERSION, _cabi.FG_F64
    E.fill_desc(d, dict(inputs, **E.host_state(state)), scalars)
    lib = _cabi.load()
    h = C.c_void_p()
    rc = lib.fg_dpop_create(C.byref(d), C.byref(h))
    msg = (lib.fg_dpop_last_error(h) or b"").decode()
    lib.fg_dpop_destroy(h)
    assert rc == _cabi.FG_ERR_ARG and "separator of 33 variables" in msg, (rc, msg)


# ---------------------------------------------------------------------------------------------------------------
# Solution cost (fg_solution_cost: k_cost_factors / k_cost_unary, warp shuffle + atomicAdd in f64)
def _engines(L, precision):
    from pydcop_b200.engine import DsaEngine, GdbaEngine, MaxSumEngine, Mgm2Engine, MgmEngine
    for cls in (MaxSumEngine, DsaEngine, MgmEngine, Mgm2Engine, GdbaEngine):
        yield cls.FAMILY, cls(L, precision=precision)


def _device_cost(eng, L, value, infinity, unary):
    import torch
    idx = torch.from_numpy(np.asarray(value, dtype=np.int32)[L.var_order]).to(eng.device)
    out = eng._solution_cost(idx, infinity, unary).cpu().numpy()
    return float(out[0]), int(out[1])


def _check_cost(inst, L, eng, value, infinity, unary=True):
    """Device (cost, violations) against the exact sum of the same terms: an f64 sum of N terms in any order is
    within (N - 1) 2^-53 sum|t| of it."""
    from pydcop_b200 import solve as S
    dcop = types.SimpleNamespace(arrays=oracle_instance(inst, L))
    if not unary:
        dcop.arrays["unary"] = np.zeros_like(inst["unary"])
    t_fac, t_var = LM.cost_terms(dcop.arrays, value)
    terms = np.concatenate([t_fac, t_var])
    hard = terms == infinity
    ok = terms[~hard]
    cost, viol = _device_cost(eng, L, value, infinity, inst["unary"] if unary else None)
    want_viol, want_cost = S.solution_cost(dcop, value, infinity)
    assert viol == want_viol == int(hard.sum())
    bound = max(len(ok) - 1, 0) * 2.0 ** -53 * float(np.abs(ok).sum())
    assert abs(cost - math.fsum(ok)) <= bound, (cost, math.fsum(ok), bound)
    assert abs(want_cost - math.fsum(ok)) <= bound
    return viol


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", ["arity8_d3", "d256", "doms_1_3_256"])
def test_solution_cost_at_the_limits(case, precision):
    inst = LM.MAXSUM[case]()
    L = build_layout(**inst)
    rng = np.random.default_rng(3)
    for fam, eng in _engines(L, precision):
        if fam == "maxsum":
            assert set(eng.kernel_plan()) == {"tiled_rt"} or case != "d256"
        for _ in range(3):
            value = (rng.integers(0, 1 << 30, L.n_vars) % inst["dom_size"]).astype(np.int32)
            _check_cost(inst, L, eng, value, float("inf"))
        eng.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_solution_cost_of_a_million_float_terms(precision):
    """10^6 mixed-sign float constraints over 7 orders of magnitude and some entries equal to `infinity`."""
    inst = LM.big_float_instance()
    L = build_layout(**inst)
    rng = np.random.default_rng(4)
    value = rng.integers(0, 3, L.n_vars).astype(np.int32)
    for fam, eng in _engines(L, precision):
        viol = _check_cost(inst, L, eng, value, 1000.0, unary=False)
        assert viol > 100
        eng.close()


@pytest.mark.parametrize("cache", ["1", "0"])
@pytest.mark.parametrize("variant", ["B", "C"])
def test_adsa_ties_on_the_binary_fast_paths(monkeypatch, variant, cache):
    """A-DSA with integer costs on the oriented-table kernels (k_dsa_step_cached, and k_dsa_step_bin without the
    active-row array): at delta == 0 the current value need not be one of the best once the variables' own costs
    are added, and then no value is dropped from the draw."""
    from pydcop_b200 import DsaEngine
    monkeypatch.setenv("PYDCOP_B200_DSA_CACHE", cache)
    inst = LM.random_graph(3000, [10], [(2, 7000)], seed=16, levels=3)
    L = build_layout(**inst)
    kw = dict(mode="min", variant=variant, seed=9, probability=0.7, var_costs=True)
    o = orc.DsaOracle(oracle_instance(inst, L), np.float32, **kw).init()
    eng = DsaEngine(L, precision="f32", **kw).init()
    assert eng.tables_or is not None and eng.row_cache is not None
    for k in range(1, 11):
        o.step()
        eng.step()
        assert np.array_equal(eng.values(), o.val), k
