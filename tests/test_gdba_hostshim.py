"""The GDBA CUDA kernel SOURCE executed on the CPU (tests/hostshim/gdba_host.cpp compiles
pydcop_b200/csrc/gdba_kernels.cuh with g++ and loops over the threads) with exactly the arrays
GdbaEngine uploads, against the reference trajectories (tests/golden/gdba_*.npz) and the oracle.
This checks the kernels' logic and the host-side array preparation without a GPU; the device run is
tests/test_gpu_zz_gdba.py's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _gdba_oracle import GdbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import (_class_array, fill_desc, fill_header, gdba_host_arrays, gdba_modifiers_view,
                                gdba_plan, host_state, mgm_host_arrays)
from pydcop_b200.layout import layout_from_instance
from test_gdba_cpu import check_trajectory
from test_mgm2_hostshim import random_mgm2_instance

SHIM_SRC = os.path.join(ROOT, "tests", "hostshim", "gdba_host.cpp")
SHIM_SO = os.path.join(ROOT, "tests", "hostshim", "_build", "gdba_host.so")
P = C.c_void_p


@pytest.fixture(scope="module")
def shim():
    deps = [SHIM_SRC, os.path.join(ROOT, "include", "pydcop_b200.h")] + [
        os.path.join(ROOT, "pydcop_b200", "csrc", f) for f in ("gdba_kernels.cuh", "mgm_kernels.cuh", "philox.cuh")]
    if not os.path.exists(SHIM_SO) or any(os.path.getmtime(d) > os.path.getmtime(SHIM_SO) for d in deps):
        os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SHIM_SO,
                        SHIM_SRC], check=True, capture_output=True)
    lib = C.CDLL(SHIM_SO)
    lib.gdba_host_cycle.argtypes = [P, C.c_int64]
    return lib


class HostGdba:
    """GdbaEngine's plan (gdba_plan) and driving API over the host-shimmed kernels."""

    def __init__(self, lib, layout, precision="f64", mode="min", modifier="A", violation="NZ", increase_mode="E",
                 stop_cycle=0, seed=0, var_rank=None, **_):
        self.lib, self.L = lib, layout
        inputs, state, scalars = gdba_plan(layout, precision, mode, modifier, violation, increase_mode, stop_cycle,
                                           seed, var_rank)
        self.has_nbr = np.diff(inputs["nbr_ptr"]) > 0
        self.gh = gdba_host_arrays(layout, inputs["nbr_ptr"], increase_mode, violation)
        self.base_mod, self.increase_mode = (0 if modifier == "A" else 1), increase_mode
        self.k = dict(inputs, **host_state(state))
        self.value = self.k["value"]
        self.classes = _class_array(layout)
        self.d = fill_desc(fill_header(_cabi.FgGdbaDesc(), precision, layout, self.classes), self.k, scalars)
        self.stop_cycle, self.cycle = scalars["stop_cycle"], 0

    @property
    def finished(self):
        return bool(self.stop_cycle and self.cycle + 1 >= self.stop_cycle)

    def init(self):
        self.lib.gdba_host_init(C.byref(self.d))
        self.cycle = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.lib.gdba_host_cycle(C.byref(self.d), self.cycle)
            self.cycle += 1
        return self

    def values(self):
        L, k = self.L, self.k
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return L.vars_to_canonical(self.value[self.cycle % 2][:L.n_vars].copy()), L.vars_to_canonical(cost)

    def modifiers(self):
        return gdba_modifiers_view(self.gh, self.k["mod"], self.base_mod, self.increase_mode)

    def record(self):
        L, k, n = self.L, self.k, self.L.n_vars
        conn = self.has_nbr[:n]
        viol = np.zeros(L.n_edges, dtype=np.uint8)
        viol[self.gh["canon_slot"]] = k["violated"][:L.n_edges]
        return dict(improve=L.vars_to_canonical(np.where(conn, k["improve"][:n].astype(np.float64), np.nan)),
                    new_value=L.vars_to_canonical(np.where(conn, k["new_value"][:n], -1).astype(np.int32)),
                    violated=viol, breakout=L.vars_to_canonical(k["breakout"][:n].copy()),
                    modifiers=self.modifiers())


def compare_with_oracle(eng, o, dt, n_cycles):
    """Every array of every round bit-identical to the oracle in the same precision."""
    assert np.array_equal(eng.values()[0], o.values()[0])
    for k in range(1, n_cycles + 1):
        o.step()
        eng.step()
        got, want = eng.record(), o.record()
        for key in want:
            if key == "improve":
                assert np.array_equal(got[key].astype(dt), want[key].astype(dt), equal_nan=True), (k, key)
            else:
                assert np.array_equal(got[key], want[key]), (k, key)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k


@pytest.mark.parametrize("name", golden_names("gdba_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_fixture(shim, name, precision):
    """f64 against the reference's trajectory; f32 against the f32 oracle (float fixtures round
    differently in f32) and, for integer costs, against the trajectory as well."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostGdba(shim, layout_from_instance(inst), precision=precision, mode=meta["mode"], seed=meta["seed"],
                   var_rank=inst["var_rank"], **meta["params"]).init()
    if precision == "f64" or "float" not in name:
        check_trajectory(eng, inst, meta, dt, name)
    else:
        o = GdbaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
        compare_with_oracle(eng, o, dt, meta["n_cycles"])


def random_gdba_instance(n, d, seed, levels=0):
    """Mixed-arity random graph (binary, ternary, unary constraints) with float or integer tables,
    variable costs, random name ranks and some initial values; sparse enough that some variables have
    one neighbour or one ternary constraint (spanning constraints)."""
    inst = random_mgm2_instance(n, d, [2, 3, 1], seed=seed, n_factors=n // 3, levels=levels)
    rng = np.random.default_rng(seed + 100)
    inst["unary"] = np.floor(rng.uniform(0, 4, int(np.sum(inst["dom_size"])))) / 4.0
    return inst


MODE_GRID = [("A", "E"), ("A", "R"), ("A", "C"), ("A", "T"), ("M", "E"), ("M", "R"), ("M", "C"), ("M", "T")]


@pytest.mark.parametrize("modifier,increase_mode", MODE_GRID)
@pytest.mark.parametrize("precision,mode,violation,levels", [("f64", "min", "NZ", 0), ("f32", "max", "NM", 3),
                                                             ("f32", "min", "MX", 3)])
def test_kernel_source_matches_oracle_on_random_graphs(shim, modifier, increase_mode, precision, mode, violation,
                                                       levels):
    inst = random_gdba_instance(400, 3, seed=13, levels=levels)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, modifier=modifier, violation=violation, increase_mode=increase_mode, seed=5)
    o = GdbaOracle(inst, dt, **kw).init()
    eng = HostGdba(shim, layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    compare_with_oracle(eng, o, dt, 8)
    assert o.stats["breakouts"] > 0
    if increase_mode != "T":
        assert o.stats["span_increases"] > 0


def test_modifier_storage_sizes():
    """T keeps one count per slot; E / R / C a table only for slots whose constraint spans the
    variable's neighbourhood (none on a binary graph of degree > 1)."""
    from pydcop_b200.generators import random_factor_graph
    inst = random_gdba_instance(300, 3, seed=2)
    L = layout_from_instance(inst)
    h = mgm_host_arrays(L)
    o = GdbaOracle(inst)
    assert gdba_host_arrays(L, h["nbr_ptr"], "T")["mod_size"] == L.n_edges
    want = sum(o.tsize[f] for v in range(o.V) for k, f in enumerate(o.cons[v]) if o.span[v][k])
    for mode in "ERC":
        g = gdba_host_arrays(L, h["nbr_ptr"], mode)
        assert g["mod_size"] == want > 0
        assert (g["mod_off"] >= 0).sum() == sum(map(sum, o.span))
    L = layout_from_instance(random_factor_graph(500, 4, 1500, 2, seed=3))
    h = mgm_host_arrays(L)
    deg = np.diff(h["nbr_ptr"])
    spanning = int(np.sum(np.repeat(deg, np.diff(L.var_ptr)) == 1))   # a degree-1 variable's binary constraints span
    assert gdba_host_arrays(L, h["nbr_ptr"], "E")["mod_size"] == 16 * spanning


def test_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu",'
                   ' sizeof(fg_gdba_desc_t), offsetof(fg_gdba_desc_t, mod_size), offsetof(fg_gdba_desc_t, dev_mod_off));'
                   'return 0;}\n' % os.path.join(ROOT, "include", "pydcop_b200.h"))
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = _cabi.FgGdbaDesc
    assert out == [C.sizeof(D), D.mod_size.offset, D.dev_mod_off.offset]


def test_descriptor_validation():
    """fg_gdba_create refuses a bad descriptor with FG_ERR_ARG and a message, and without a device reports
    FG_ERR_CUDA — never a CPU path."""
    import torch
    lib = _cabi.load()
    inst = random_gdba_instance(60, 3, seed=1)
    d = HostGdba(None, layout_from_instance(inst), violation="NM").d

    def create():
        h = P()
        rc = lib.fg_gdba_create(C.byref(d), C.byref(h))
        msg = (lib.fg_gdba_last_error(h) or b"").decode()
        lib.fg_gdba_destroy(h)
        return rc, msg

    for field, bad, word in (("modifier", 2, "modifier"), ("violation", 3, "violation"),
                             ("increase_mode", 4, "increase_mode"), ("stop_cycle", -1, "stop_cycle")):
        good = getattr(d, field)
        setattr(d, field, bad)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and word in msg, (field, msg)
        setattr(d, field, good)
    for field in ("dev_viol_ref", "dev_mod_off", "dev_improve"):
        good = getattr(d, field)
        setattr(d, field, None)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and "missing" in msg, field
        setattr(d, field, good)
    d.increase_mode, d.mod_size = _cabi.GDBA_INCREASE_MODES["T"], 1
    rc, msg = create()
    assert rc == _cabi.FG_ERR_ARG and "mod_size" in msg
    d.mod_size = d.n_edges
    if not torch.cuda.is_available():
        rc, msg = create()
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device" in msg


def test_kernel_source_isolated_variables(shim):
    """A variable without neighbours keeps optimal_cost_value over its own costs: here the unary
    constraint is NOT part of it (gdba.py:304-315)."""
    from test_mgm2_cpu import unit_instance
    inst = unit_instance([list(range(3))], [([0], lambda x: 5 - x)])
    inst["unary"] = np.array([1.0, 0.5, 0.5])
    for precision, mode, want in (("f64", "min", 1), ("f32", "max", 0)):
        eng = HostGdba(shim, layout_from_instance(inst), precision=precision, mode=mode).init().step(3)
        val, cost = eng.values()
        assert val.tolist() == [want] and cost.tolist() == [inst["unary"][want]]
        o = GdbaOracle(inst, mode=mode).init().step(3)
        assert o.values()[0].tolist() == [want]


@pytest.mark.parametrize("modifier,increase_mode", LM.GDBA_MODES)
@pytest.mark.parametrize("case", list(LM.LOCAL))
def test_kernel_source_at_the_limits(shim, case, modifier, increase_mode):
    """Domain sizes 1 and 256 and the mix {1, 2, 256} (tests/_limits.py), as tests/test_gpu_limits.py runs them."""
    inst = LM.gdba_instance(case)
    kw = dict(mode="min", modifier=modifier, violation="NZ", increase_mode=increase_mode, seed=23)
    o = GdbaOracle(inst, np.float64, **kw).init()
    eng = HostGdba(shim, layout_from_instance(inst), precision="f64", var_rank=inst["var_rank"], **kw).init()
    compare_with_oracle(eng, o, np.float64, 6)
    assert o.stats["breakouts"] > 0
