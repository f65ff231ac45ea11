"""The generic DSA CUDA kernel SOURCE (pydcop_b200/csrc/dsa_generic.cuh, unmodified) on the CPU
through tests/hostshim/dsa_generic_host.cpp, against the reference trajectories and the oracle —
including frozen ghost variables and global Philox ids as the sharded path uses them, and arities
the GPU tests do not reach.  Needs the CUDA toolkit headers (not a GPU)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import _limits as LM
import oracle as orc
from bench import oracle_instance
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array
from pydcop_b200.layout import default_var_csr, layout_from_instance
from test_maxsum_generic_hostshim import CUDA_INC, _mixed_instance

SRC = os.path.join(ROOT, "tests", "hostshim", "dsa_generic_host.cpp")
SO = os.path.join(ROOT, "tests", "hostshim", "_build", "dsa_generic_host.so")
P = C.c_void_p

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA toolkit headers not present")


class _Host(C.Structure):
    _fields_ = [("classes", P), ("n_classes", C.c_int32), ("n_vars", C.c_int32), ("precision", C.c_int32),
                ("mode_max", C.c_int32), ("variant", C.c_int32), ("tables", P), ("dom_size", P), ("var_id", P),
                ("edge_var", P), ("edge_class", P), ("var_ptr", P), ("slot_edge", P), ("has_nbr", P), ("prob", P),
                ("con_opt", P), ("value", P * 2), ("value_cost", P), ("seed", C.c_uint64), ("var_cost", P),
                ("unary_off", P)]


def _lib():
    deps = [SRC] + [os.path.join(ROOT, "pydcop_b200", "csrc", f) for f in ("dsa_generic.cuh", "common.cuh", "philox.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-I", CUDA_INC, "-shared", "-fPIC",
                        "-o", SO, SRC], check=True, capture_output=True)
    return C.CDLL(SO)


class HostDsa:
    """What DsaEngine prepares on the host (generic path), stepped by the host-shimmed kernels."""

    def __init__(self, inst, precision="f64", mode="min", probability=0.7, p_mode="fixed", variant="B",
                 stop_cycle=0, seed=0, var_global_id=None, frozen=None, var_costs=False, **_):
        self.lib = _lib()
        self.L = L = layout_from_instance(inst)
        dt = np.float64 if precision == "f64" else np.float32
        arity = np.array([c.arity for c in L.classes], dtype=np.int64)
        n_count = np.zeros(L.n_vars, dtype=np.int64)
        if L.n_edges:
            np.add.at(n_count, L.slot_var, arity[L.edge_class[L.slot_edge]] - 1)
        has_nbr = (n_count > 0).astype(np.uint8)
        if frozen is not None:
            has_nbr[np.asarray(frozen, dtype=bool)[L.var_order]] = 0
        var_id = L.var_order if var_global_id is None else np.asarray(var_global_id, np.int32)[L.var_order]
        prob = (np.where(n_count > 0, 1.0 / np.maximum(n_count, 1) * 1.2, 0.0) if p_mode == "arity"
                else np.full(L.n_vars, float(probability)))
        iso = np.zeros(L.n_vars, dtype=np.int32)
        for v in np.nonzero(n_count == 0)[0]:
            c = L.unary[L.unary_off[v]:L.unary_off[v] + L.dom_size[v]]
            iso[v] = int(np.argmin(c)) if mode == "min" else int(len(c) - 1 - np.argmax(c[::-1]))
        c = np.ascontiguousarray
        n = max(L.n_vars, 1)
        self.keep = dict(classes=_class_array(L), tables=c(L.tables, dt), dom_size=c(L.dom_size, np.int32),
                         var_id=c(var_id, np.int32), edge_var=c(L.edge_var, np.int32),
                         edge_class=c(L.edge_class, np.int32), var_ptr=c(L.var_ptr, np.int32),
                         slot_edge=c(L.slot_edge, np.int32), has_nbr=c(has_nbr, np.uint8), prob=c(prob, np.float64),
                         con_opt=np.zeros(max(L.n_factors, 1), dt), v0=c(np.resize(iso, n), np.int32),
                         v1=np.zeros(n, np.int32), value_cost=np.zeros(n, dt),
                         var_cost=c(L.unary, dt), unary_off=c(L.unary_off, np.int64))
        h = _Host()
        k = self.keep
        for name in ("tables", "dom_size", "var_id", "edge_var", "edge_class", "var_ptr", "slot_edge", "has_nbr",
                     "prob", "con_opt", "value_cost"):
            setattr(h, name, P(k[name].ctypes.data))
        h.classes = C.cast(k["classes"], P)
        h.value[0], h.value[1] = k["v0"].ctypes.data, k["v1"].ctypes.data
        h.n_classes, h.n_vars = len(L.classes), L.n_vars
        h.precision = _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        h.mode_max, h.variant, h.seed = int(mode == "max"), _cabi.DSA_VARIANTS[variant], int(seed)
        if var_costs:      # A-DSA (adsa.py:344-377)
            h.var_cost, h.unary_off = P(k["var_cost"].ctypes.data), P(k["unary_off"].ctypes.data)
        self.h, self.cur, self.cycle, self.stop_cycle = h, 0, 0, int(stop_cycle)

    def init(self):
        self.lib.dsa_host_init(C.byref(self.h))
        self.cur, self.cycle = 0, 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.stop_cycle and self.cycle >= self.stop_cycle:
                break
            self.lib.dsa_host_step(C.byref(self.h), self.cur, C.c_uint32(self.cycle))
            self.cur ^= 1
            self.cycle += 1
        return self

    def values(self):
        return self.L.vars_to_canonical(self.keep["v%d" % self.cur][:self.L.n_vars])


@pytest.mark.parametrize("name", golden_names("dsa_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_generic_dsa_kernel_source_matches_reference_trajectory(name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    e = HostDsa(inst, precision, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            e.step()
        assert np.array_equal(e.values(), inst["value"][k]), (name, k)


@settings(max_examples=25, deadline=None)
@given(st.integers(0, 10_000), st.integers(5, 24), st.sampled_from(["A", "B", "C"]), st.sampled_from(["min", "max"]),
       st.sampled_from(["fixed", "arity"]), st.booleans())
def test_generic_dsa_kernel_source_fuzz(seed, n_vars, variant, mode, p_mode, sharded_style):
    """Arities 1-5, mixed domains, few cost levels (ties), optionally with frozen variables and
    permuted Philox ids as a shard of a larger problem would have."""
    rng = np.random.default_rng(seed)
    shapes = [(int(a), int(rng.integers(1, 8))) for a in rng.choice([1, 2, 3, 5], size=3) if a <= n_vars]
    inst = _mixed_instance(rng, n_vars, [2, 3, 4, 6], shapes)
    inst["tables"] = np.round(inst["tables"]).astype(np.float32)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n_vars, inst["edge_var"])
    kw = dict(mode=mode, variant=variant, p_mode=p_mode, probability=0.6, seed=seed + 1)
    extra = {}
    if sharded_style:
        extra = dict(var_id=rng.permutation(1000)[:n_vars].astype(np.int32), frozen=rng.random(n_vars) < 0.25)
    o = orc.DsaOracle(inst, np.float64, **kw, **extra).init()
    e = HostDsa(inst, "f64", var_global_id=extra.get("var_id"), frozen=extra.get("frozen"), **kw).init()
    live = o.has_nbr.astype(bool)
    assert np.array_equal(e.values()[live], o.val[live])
    e.keep["v0"][:] = np.asarray(o.val, np.int32)[e.L.var_order]     # frozen / isolated entries: same start
    e.keep["v1"][:] = e.keep["v0"]
    for k in range(7):
        o.step()
        e.step()
        assert np.array_equal(e.values(), o.val), k


@pytest.mark.parametrize("name", golden_names("adsa_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_generic_kernel_source_with_variable_costs_matches_reference_adsa(name, precision):
    """A-DSA = the DSA kernel with the variables' own costs added to the candidates (adsa.py:344-377): the
    trajectories recorded from the UNMODIFIED ADsaComputation under aligned ticks (oracle/make_golden_adsa.py)."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    p = meta["params"]
    e = HostDsa(inst, precision, mode=meta["mode"], seed=meta["seed"], probability=p["probability"],
                variant=p["variant"], var_costs=True).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            e.step()
        assert np.array_equal(e.values(), inst["value"][k]), k


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("case,variant,mode,var_costs", LM.DSA_RUNS)
def test_generic_dsa_kernel_source_at_the_limits(case, variant, mode, var_costs, precision):
    """The C-ABI limit instances of tests/_limits.py (domain sizes 1 and 256, all 256 values tied, arity 8, a hub
    of degree 2400), as tests/test_gpu_limits.py runs them on the device."""
    inst = LM.DSA[case]()
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, variant=variant, seed=7, probability=0.7, var_costs=var_costs)
    e = HostDsa(inst, precision, **kw).init()
    o = orc.DsaOracle(oracle_instance(inst, e.L), dt, **kw).init()
    assert np.array_equal(e.values(), o.val)
    for k in range(1, 11):
        o.step()
        e.step()
        assert np.array_equal(e.values(), o.val), k
