"""The MGM CUDA kernel SOURCE executed on the CPU (tests/hostshim/mgm_host.cpp runs
fg_mgm_init / fg_mgm_step's launch sequence from pydcop_b200/csrc/mgm_fast_kernels.cuh, thread after thread) with exactly the arrays
MgmEngine uploads, against the reference trajectories and the oracle.  This checks the kernels'
logic and the host-side array preparation without a GPU; it says nothing about the device run,
which tests/test_gpu_zz_mgm.py covers."""
import os

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _hostshim import HostRun
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200.engine import fill_desc, mgm_plan
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.layout import default_var_csr, layout_from_instance


class HostMgm(HostRun):
    """MgmEngine's plan (mgm_plan) run by tests/hostshim/mgm_host.cpp."""

    def __init__(self, layout, precision="f64", mode="min", stop_cycle=0, seed=0, var_rank=None,
                 isolated_value=None, var_global_id=None, var_seed=None, **_):
        plan = mgm_plan(layout, precision, mode, stop_cycle, seed, var_rank, isolated_value,
                        var_global_id=var_global_id, var_seed=var_seed)
        super().__init__("mgm", layout, plan, precision)
        self.keep = self.k

    def values(self):
        L, k = self.L, self.keep
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return L.vars_to_canonical(k["value"][:L.n_vars]), L.vars_to_canonical(cost)

    def gains(self):
        L, k = self.L, self.keep
        return (L.vars_to_canonical(k["gain"][:L.n_vars].astype(np.float64)),
                L.vars_to_canonical(k["new_value"][:L.n_vars]))


@pytest.mark.parametrize("name", golden_names("mgm_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_reference_trajectory(name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostMgm(layout_from_instance(inst), precision=precision, mode=meta["mode"],
                  seed=meta["seed"], var_rank=inst["var_rank"], **meta["params"]).init()
    has_nbr = ~np.isnan(inst["gain"][1])
    for k in range(meta["n_cycles"] + 1):
        ran = False
        if k:
            before = eng.cycle
            eng.step()
            ran = eng.cycle > before
        val, cost = eng.values()
        assert np.array_equal(val, inst["value"][k]), (name, k)
        known = ~np.isnan(inst["cost"][k])
        assert np.array_equal(~np.isnan(cost), known), (name, k)
        assert np.array_equal(cost[known].astype(dt), inst["cost"][k][known].astype(dt)), (name, k)
        if ran:
            gain, new_value = eng.gains()
            assert np.array_equal(gain[has_nbr].astype(dt), inst["gain"][k][has_nbr].astype(dt)), (name, k)
            assert np.array_equal(new_value[has_nbr], inst["new_value"][k][has_nbr]), (name, k)
    assert eng.cycle + 1 == int(inst["cycle_count"][-1].max())


@pytest.mark.parametrize("precision,d,arity,mode", [("f64", 10, 2, "min"), ("f32", 10, 2, "min"),
                                                    ("f64", 5, 3, "max"), ("f32", 20, 2, "min")])
def test_kernel_source_matches_oracle_with_float_costs(precision, d, arity, mode):
    """Float tables and float variable costs: the kernel keeps the oracle's operand order, so
    values, costs and gains are bit-identical in both precisions."""
    n = 3000
    inst = random_factor_graph(n, d, n * 2 if arity == 2 else n, arity, seed=3, noise=0.5, int_tables=False)
    rng = np.random.default_rng(5)
    inst["var_rank"] = rng.permutation(n).astype(np.int32)
    inst["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, d, n), -1).astype(np.int32)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    dt = np.float64 if precision == "f64" else np.float32
    o = orc.MgmOracle(inst, dt, mode=mode, seed=17).init()
    eng = HostMgm(layout_from_instance(inst), precision=precision, mode=mode, seed=17,
                  var_rank=inst["var_rank"]).init()
    assert np.array_equal(eng.values()[0], o.val)
    moved = 0
    for k in range(1, 11):
        prev = o.val.copy()
        o.step()
        eng.step()
        val, cost = eng.values()
        assert np.array_equal(val, o.val), k
        assert np.array_equal(cost.astype(dt), o.cost), k
        gain, new_value = eng.gains()
        assert np.array_equal(gain.astype(dt), o.gain) and np.array_equal(new_value, o.new_val), k
        moved += int((prev != o.val).sum())
    assert moved > 0


class HostMgmFast(HostMgm):
    """HostMgm with the oriented tables in the descriptor: the value phase runs k_mgm_gain_bin, as MgmEngine's."""

    def __init__(self, layout, precision, chunk, mode="min", **kw):
        import torch
        from pydcop_b200.engine import dsa_fast_arrays
        super().__init__(layout, precision=precision, mode=mode, **kw)
        dt = np.float64 if precision == "f64" else np.float32
        fast = dsa_fast_arrays(layout, torch.from_numpy(np.ascontiguousarray(layout.tables, dtype=dt)), mode)
        assert fast is not None
        tables_or, slot_tab, slot_nbr, _, D = fast
        self.fkeep = dict(slot_nbr=np.ascontiguousarray(slot_nbr.numpy(), np.int32),
                          slot_tab=np.ascontiguousarray(slot_tab.numpy(), np.int64),
                          tables_or=np.ascontiguousarray(tables_or.numpy(), dt))
        fill_desc(self.d, self.fkeep, dict(fast_dom=D, fast_chunk=chunk))


@pytest.mark.parametrize("d,mode,precision,chunk", [(4, "min", "f64", 4), (8, "max", "f32", 2), (10, "min", "f32", 4),
                                                    (16, "min", "f64", 2), (20, "min", "f32", 4), (20, "max", "f64", 4)])
def test_fast_value_phase_source_matches_generic_and_oracle(d, mode, precision, chunk):
    n = 2500
    inst = random_factor_graph(n, d, int(n * 2.7), 2, seed=d + 1, noise=0.5, int_tables=False)
    rng = np.random.default_rng(d)
    inst["var_rank"] = rng.permutation(n).astype(np.int32)
    inst["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, d, n), -1).astype(np.int32)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    dt = np.float64 if precision == "f64" else np.float32
    L = layout_from_instance(inst)
    o = orc.MgmOracle(inst, dt, mode=mode, seed=23).init()
    fast = HostMgmFast(L, precision, chunk, mode=mode, seed=23, var_rank=inst["var_rank"]).init()
    slow = HostMgm(L, precision=precision, mode=mode, seed=23, var_rank=inst["var_rank"]).init()
    moved = 0
    for k in range(1, 10):
        prev = o.val.copy()
        o.step()
        fast.step()
        slow.step()
        for e in (fast, slow):
            val, cost = e.values()
            assert np.array_equal(val, o.val), k
            assert np.array_equal(cost.astype(dt), o.cost), k
            gain, new_value = e.gains()
            assert np.array_equal(gain.astype(dt), o.gain) and np.array_equal(new_value, o.new_val), k
        moved += int((prev != o.val).sum())
    assert moved > 0 and np.diff(inst["var_ptr"]).max() > 2 * chunk


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("case", list(LM.MGM))
def test_kernel_source_at_the_limits(case, precision, mode):
    """Domain sizes 1 and 256 with every value tied (tests/_limits.py), as tests/test_gpu_limits.py runs them."""
    inst = LM.MGM[case]()
    dt = np.float64 if precision == "f64" else np.float32
    o = orc.MgmOracle(inst, dt, mode=mode, seed=17).init()
    eng = HostMgm(layout_from_instance(inst), precision=precision, mode=mode, seed=17,
                  var_rank=inst["var_rank"]).init()
    assert np.array_equal(eng.values()[0], o.val)
    for k in range(1, 9):
        o.step()
        eng.step()
        val, cost = eng.values()
        assert np.array_equal(val, o.val), k
        assert np.array_equal(cost.astype(dt), o.cost, equal_nan=True), k
        gain, new_value = eng.gains()
        assert np.array_equal(gain.astype(dt), o.gain) and np.array_equal(new_value, o.new_val), k
