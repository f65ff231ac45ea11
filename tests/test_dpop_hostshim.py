"""The DPOP CUDA kernel SOURCE executed on the CPU (tests/hostshim/dpop_host.cpp compiles
pydcop_b200/csrc/dpop_kernels.cuh with g++ and walks the schedule) with the descriptor DpopEngine builds,
against the reference's messages (tests/golden/dpop_*.npz) and the oracle.  This checks the per-entry and
per-node device functions and the host-side descriptors without a GPU; the device run is
tests/test_gpu_zz_dpop.py's."""
import ctypes as C

import numpy as np
import pytest

import _hostshim as hs
from _dpop_oracle import DpopOracle
import _limits as LM
from pydcop_b200 import _cabi, pseudotree as pt
from pydcop_b200.engine import dpop_plan, fill_desc, host_state
from pydcop_b200.layout import build_layout
from test_dpop_cpu import NAMES, _integer_without_sentinel, check_against_golden, load, same, tree_of



@pytest.fixture(scope="module")
def shim():
    lib = hs.build("dpop_host")
    lib.dpop_host_run.argtypes = [C.c_void_p]
    return lib


class HostDpop:
    """DpopEngine's plan (dpop_plan) with host arrays, run through the shim."""

    def __init__(self, lib, inst, tree, precision, mode):
        L = build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"], unary=inst["unary"])
        inputs, state, scalars = dpop_plan(L, tree, pt.schedule(tree), precision, mode)
        self.util_off = inputs["util_off"]
        self.k = k = dict(inputs, **host_state(state))
        d = _cabi.FgDpopDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        fill_desc(d, k, scalars)
        lib.dpop_host_run(C.byref(d))
        n = L.n_vars
        self.value, self.cost = k["value"][:n], k["cost"][:n].astype(np.float64)
        self.unresolved = int(k["unresolved"][0])

    def util(self, tree, u):
        off = self.util_off[u]
        return self.k["arena"][off:off + tree.util_size[u]].reshape(
            tuple(int(self.k["dom_size"][v]) for v in tree.sep[u]))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_shim_matches_fixture_and_oracle(shim, name, precision):
    inst, meta = load(name)
    dt = np.float64 if precision == "f64" else np.float32
    t = tree_of(inst)
    h = HostDpop(shim, inst, t, precision, meta["mode"])
    if precision == "f64" or _integer_without_sentinel(inst):
        check_against_golden(inst, meta, t, lambda u: h.util(t, u), h.value, h.cost, dt)
    o = DpopOracle(inst, t, dt, meta["mode"]).run()
    for u in range(t.n_vars):
        assert same(h.util(t, u), o.util[u]), u
    assert np.array_equal(h.value, o.value) and same(h.cost, np.asarray(o.cost, dtype=dt))
    assert h.unresolved == o.unresolved and (h.unresolved > 0) == (meta["error"] == "IndexError")


def test_shim_runs_big_and_light_nodes_like_the_oracle(shim):
    """A chain with separators of 4 at d = 10 (UTIL of 10^4 entries: grid-wide nodes) under light pendant
    leaves, float costs, max mode."""
    from pydcop_b200.generators import bounded_separator_instance
    inst = bounded_separator_instance(14, 10, back=3, span=1, seed=6, float_costs=True)
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    assert pt.schedule(t).big_nodes
    h = HostDpop(shim, inst, t, "f64", "max")
    o = DpopOracle(inst, t, np.float64, "max").run()
    for u in range(t.n_vars):
        assert same(h.util(t, u), o.util[u]), u
    assert np.array_equal(h.value, o.value) and same(h.cost, o.cost)


@pytest.mark.parametrize("precision,mode", [("f64", "min"), ("f32", "max")])
@pytest.mark.parametrize("case", ["d256", "domain_one", "separator_32"])
def test_shim_at_the_limits(shim, case, precision, mode):
    """tests/_limits.py's DPOP instances: UTIL tables of 256^2 entries, variables with one value, and a separator
    of FG_DPOP_MAX_SEP = 32 variables."""
    inst = {"d256": LM.dpop_d256, "domain_one": LM.dpop_with_domain_one, "separator_32": lambda: LM.clique(33)}[case]()
    dt = np.float64 if precision == "f64" else np.float32
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    h = HostDpop(shim, inst, t, precision, mode)
    o = DpopOracle(inst, t, dt, mode).run()
    for u in range(t.n_vars):
        assert same(h.util(t, u), o.util[u]), u
    assert np.array_equal(h.value, o.value) and same(h.cost, np.asarray(o.cost, dtype=dt))
    assert h.unresolved == o.unresolved == 0
