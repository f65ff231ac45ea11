"""The generic DSA CUDA kernel SOURCE (pydcop_b200/csrc/dsa_generic.cuh, unmodified) on the CPU
through tests/hostshim/dsa_generic_host.cpp, against the reference trajectories and the oracle —
including frozen ghost variables and global Philox ids as the sharded path uses them, and arities
the GPU tests do not reach.  Needs the CUDA toolkit headers (not a GPU)."""
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import _limits as LM
import oracle as orc
from _hostshim import CUDA_INC, HostRun
from bench import oracle_instance
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200.engine import dsa_plan
from pydcop_b200.layout import default_var_csr, layout_from_instance
from test_maxsum_generic_hostshim import _mixed_instance

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA toolkit headers not present")


class HostDsa(HostRun):
    """DsaEngine's plan (dsa_plan) run by tests/hostshim/dsa_generic_host.cpp: the generic kernels."""

    def __init__(self, inst, precision="f64", mode="min", probability=0.7, p_mode="fixed", variant="B",
                 stop_cycle=0, seed=0, var_global_id=None, frozen=None, var_costs=False, var_seed=None, **_):
        L = layout_from_instance(inst)
        super().__init__("dsa", L, dsa_plan(L, precision, mode, probability, p_mode, variant, stop_cycle, seed,
                                            var_global_id=var_global_id, frozen=frozen, var_costs=var_costs,
                                            var_seed=var_seed), precision)

    def values(self):
        return self.L.vars_to_canonical(self.value[:self.L.n_vars].copy())


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
    e.k["value"][0][:] = np.asarray(o.val, np.int32)[e.L.var_order]     # frozen / isolated entries: same start
    e.k["value"][1][:] = e.k["value"][0]
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
