"""The MGM CUDA kernel SOURCE executed on the CPU (tests/hostshim/mgm_host.cpp compiles
pydcop_b200/csrc/mgm_kernels.cuh with g++ and loops over the threads) with exactly the arrays
MgmEngine uploads, against the reference trajectories and the oracle.  This checks the kernels'
logic and the host-side array preparation without a GPU; it says nothing about the device run,
which tests/test_gpu_zz_mgm.py covers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array, fill_desc, host_state, mgm_plan
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.layout import default_var_csr, layout_from_instance

SHIM_SRC = os.path.join(ROOT, "tests", "hostshim", "mgm_host.cpp")
SHIM_SO = os.path.join(ROOT, "tests", "hostshim", "_build", "mgm_host.so")
P = C.c_void_p


class _Arrays(C.Structure):
    _fields_ = [("classes", P), ("dom_size", P), ("var_id", P), ("var_rank", P), ("edge_var", P),
                ("edge_class", P), ("var_ptr", P), ("slot_edge", P), ("nbr_ptr", P), ("nbr_idx", P),
                ("unary_off", P), ("init_value", P), ("tables", P), ("unary", P), ("value", P),
                ("cost", P), ("has_cost", P), ("gain", P), ("new_value", P),
                ("n_vars", C.c_int32), ("precision", C.c_int32), ("mode_max", C.c_int32),
                ("seed", C.c_uint64)]


@pytest.fixture(scope="module")
def shim():
    deps = [SHIM_SRC, os.path.join(ROOT, "pydcop_b200", "csrc", "mgm_kernels.cuh"),
            os.path.join(ROOT, "pydcop_b200", "csrc", "philox.cuh"),
            os.path.join(ROOT, "pydcop_b200", "csrc", "mgm_fast_kernels.cuh"),
            os.path.join(ROOT, "pydcop_b200", "csrc", "row_load.cuh"),
            os.path.join(ROOT, "include", "pydcop_b200.h")]
    if not os.path.exists(SHIM_SO) or any(os.path.getmtime(d) > os.path.getmtime(SHIM_SO) for d in deps):
        os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SHIM_SO,
                        SHIM_SRC], check=True, capture_output=True)
    return C.CDLL(SHIM_SO)


class HostMgm:
    """MgmEngine's plan (mgm_plan) and driving API over the host-shimmed kernels."""

    def __init__(self, lib, layout, precision="f64", mode="min", stop_cycle=0, seed=0, var_rank=None,
                 isolated_value=None, **_):
        self.lib, self.L = lib, layout
        inputs, state, scalars = mgm_plan(layout, precision, mode, stop_cycle, seed, var_rank, isolated_value)
        self.classes = _class_array(layout)
        self.keep = dict(inputs, **host_state(state))
        a = fill_desc(_Arrays(), self.keep, {k: scalars[k] for k in ("mode_max", "seed")}, prefix="")
        a.classes = C.cast(self.classes, P)
        a.n_vars, a.precision = layout.n_vars, _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        self.a, self.stop_cycle, self.cycle = a, int(stop_cycle), 0

    @property
    def finished(self):
        return bool(self.stop_cycle and self.cycle + 1 >= self.stop_cycle)

    def init(self):
        self.lib.mgm_host_init(C.byref(self.a))
        self.cycle = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.lib.mgm_host_cycle(C.byref(self.a), C.c_uint32(self.cycle + 1))
            self.cycle += 1
        return self

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
def test_kernel_source_matches_reference_trajectory(shim, name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostMgm(shim, layout_from_instance(inst), precision=precision, mode=meta["mode"],
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
def test_kernel_source_matches_oracle_with_float_costs(shim, precision, d, arity, mode):
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
    eng = HostMgm(shim, layout_from_instance(inst), precision=precision, mode=mode, seed=17,
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


class _Fast(C.Structure):
    _fields_ = [("slot_nbr", P), ("slot_tab", P), ("tables_or", P), ("dom", C.c_int32), ("chunk", C.c_int32)]


class HostMgmFast(HostMgm):
    """HostMgm stepping the FAST value-phase kernel on the DSA fast-path arrays."""

    def __init__(self, lib, layout, precision, chunk, mode="min", **kw):
        import torch
        from pydcop_b200.engine import dsa_fast_arrays
        super().__init__(lib, layout, precision=precision, mode=mode, **kw)
        dt = np.float64 if precision == "f64" else np.float32
        fast = dsa_fast_arrays(layout, torch.from_numpy(np.ascontiguousarray(layout.tables, dtype=dt)), mode)
        assert fast is not None
        tables_or, slot_tab, slot_nbr, _, D = fast
        self.fkeep = dict(slot_nbr=np.ascontiguousarray(slot_nbr.numpy(), np.int32),
                          slot_tab=np.ascontiguousarray(slot_tab.numpy(), np.int64),
                          tables_or=np.ascontiguousarray(tables_or.numpy(), dt))
        self.f = _Fast(P(self.fkeep["slot_nbr"].ctypes.data), P(self.fkeep["slot_tab"].ctypes.data),
                       P(self.fkeep["tables_or"].ctypes.data), D, chunk)

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            assert self.lib.mgm_host_cycle_fast(C.byref(self.a), C.byref(self.f), C.c_uint32(self.cycle + 1)) == 0
            self.cycle += 1
        return self


@pytest.mark.parametrize("d,mode,precision,chunk", [(4, "min", "f64", 4), (8, "max", "f32", 2), (10, "min", "f32", 4),
                                                    (16, "min", "f64", 2), (20, "min", "f32", 4), (20, "max", "f64", 4)])
def test_fast_value_phase_source_matches_generic_and_oracle(shim, d, mode, precision, chunk):
    n = 2500
    inst = random_factor_graph(n, d, int(n * 2.7), 2, seed=d + 1, noise=0.5, int_tables=False)
    rng = np.random.default_rng(d)
    inst["var_rank"] = rng.permutation(n).astype(np.int32)
    inst["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, d, n), -1).astype(np.int32)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    dt = np.float64 if precision == "f64" else np.float32
    L = layout_from_instance(inst)
    o = orc.MgmOracle(inst, dt, mode=mode, seed=23).init()
    fast = HostMgmFast(shim, L, precision, chunk, mode=mode, seed=23, var_rank=inst["var_rank"]).init()
    slow = HostMgm(shim, L, precision=precision, mode=mode, seed=23, var_rank=inst["var_rank"]).init()
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
def test_kernel_source_at_the_limits(shim, case, precision, mode):
    """Domain sizes 1 and 256 with every value tied (tests/_limits.py), as tests/test_gpu_limits.py runs them."""
    inst = LM.MGM[case]()
    dt = np.float64 if precision == "f64" else np.float32
    o = orc.MgmOracle(inst, dt, mode=mode, seed=17).init()
    eng = HostMgm(shim, layout_from_instance(inst), precision=precision, mode=mode, seed=17,
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
