"""CPU: size-independent properties of the oracle (and therefore of the path it pins), and a
regeneration check of the committed fixtures against the live reference."""
import os
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import oracle as orc
import ref_shim
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.layout import default_var_csr


def _inst(n_vars, d, n_factors, arity, seed):
    inst = random_factor_graph(n_vars, d, n_factors, arity, seed=seed, int_tables=False)
    vp, ve = default_var_csr(n_vars, inst["edge_var"])
    return dict(inst, var_ptr=vp, var_edge=ve)


@settings(max_examples=25, deadline=None)
@given(st.integers(3, 30), st.integers(2, 6), st.integers(1, 40), st.sampled_from([1, 2, 3]),
       st.integers(0, 10_000), st.sampled_from(["both", "vars", "factors", "none"]),
       st.sampled_from(["leafs", "leafs_vars", "all"]))
def test_negation_symmetry(n_vars, d, n_factors, arity, seed, damping_nodes, start):
    """max-mode on negated costs mirrors min-mode exactly (every IEEE op commutes with negation)."""
    arity = min(arity, n_vars)
    inst = _inst(n_vars, d, n_factors, arity, seed)
    neg = dict(inst, tables=-inst["tables"], unary=-inst["unary"])
    kw = dict(damping_nodes=damping_nodes, start_messages=start)
    a = orc.MaxSumOracle(inst, np.float64, mode="min", **kw).init().step(12)
    b = orc.MaxSumOracle(neg, np.float64, mode="max", **kw).init().step(12)
    assert np.array_equal(a.q, -b.q) and np.array_equal(a.r, -b.r)
    assert np.array_equal(a.value, b.value)
    assert np.array_equal(a.q_sent, b.q_sent) and np.array_equal(a.r_sent, b.r_sent)


@settings(max_examples=15, deadline=None)
@given(st.integers(4, 25), st.integers(2, 5), st.integers(2, 30), st.integers(0, 10_000))
def test_factor_order_does_not_matter_when_links_are_kept(n_vars, d, n_factors, seed):
    """Permuting the factors (and keeping every variable's `links` order) permutes the messages."""
    inst = _inst(n_vars, d, n_factors, 2, seed)
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n_factors)                      # new position -> old factor
    ev = inst["edge_var"].reshape(n_factors, 2)[perm].reshape(-1)
    tb = inst["tables"].reshape(n_factors, d * d)[perm].reshape(-1)
    old_edge_of_new = (perm[:, None] * 2 + np.arange(2)[None, :]).reshape(-1)   # new edge -> old edge
    new_of_old = np.empty_like(old_edge_of_new)
    new_of_old[old_edge_of_new] = np.arange(len(old_edge_of_new))
    p = dict(inst, edge_var=ev, tables=tb, var_edge=new_of_old[inst["var_edge"]].astype(np.int32))
    a = orc.MaxSumOracle(inst, np.float64).init().step(10)
    b = orc.MaxSumOracle(p, np.float64).init().step(10)
    idx = (old_edge_of_new[:, None] * d + np.arange(d)[None, :]).reshape(-1)    # new element -> old element
    assert np.array_equal(b.q, a.q[idx]) and np.array_equal(b.r, a.r[idx])
    assert np.array_equal(a.value, b.value)


@settings(max_examples=15, deadline=None)
@given(st.integers(3, 40), st.integers(2, 6), st.integers(1, 60), st.integers(0, 10_000),
       st.sampled_from(["A", "B", "C"]))
def test_dsa_is_a_pure_function_of_the_seed(n_vars, d, n_factors, seed, variant):
    inst = _inst(n_vars, d, n_factors, 2, seed)
    inst["tables"] = np.round(inst["tables"])       # ties
    a = orc.DsaOracle(inst, np.float64, variant=variant, seed=seed).init().step(10)
    b = orc.DsaOracle(inst, np.float64, variant=variant, seed=seed).init().step(10)
    c = orc.DsaOracle(inst, np.float64, variant=variant, seed=seed + 1).init().step(10)
    assert np.array_equal(a.val, b.val)
    assert a.val.shape == c.val.shape
    # costs never get worse in expectation is NOT asserted (DSA is stochastic); only determinism is


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
def test_fixtures_regenerate_bit_for_bit(tmp_path):
    """oracle/make_golden.py, re-run now against the live reference, reproduces the committed
    message trajectories and values (the only run-to-run freedom is the summation order of the
    reported selection cost, see test_oracle_golden.py)."""
    code = (
        "import sys, os; sys.path.insert(0, %r); sys.argv = ['make_golden.py', 'ms_arity3_d4', 'dsa_A', 'ms_tree_leafs']\n"
        "import make_golden as m; m.GOLDEN = %r; m.main()\n") % (os.path.join(ROOT, "oracle"), str(tmp_path))
    subprocess.run([sys.executable, "-W", "ignore", "-c", code], check=True, capture_output=True, timeout=300)
    # (the YAML-loaded instances are left out: the reference's loader does not fix the constraint
    # order across interpreter runs, so their edges may come out permuted)
    for name, keys in (("ms_arity3_d4", ("r_state", "q_state", "r_sent", "q_sent", "value", "unary")),
                       ("ms_tree_leafs", ("r_state", "q_state", "r_sent", "q_sent", "value")),
                       ("dsa_A", ("value", "cycle_count"))):
        new = np.load(os.path.join(str(tmp_path), name + ".npz"))
        old = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        for k in keys:
            assert np.array_equal(new[k], old[k]), (name, k)


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
def test_mgm_fixtures_regenerate_bit_for_bit(tmp_path):
    """oracle/make_golden_mgm.py re-run against the live reference reproduces the committed MGM
    trajectories, including the one with variable costs (whose sums the reference accumulates in a
    set's iteration order — exact for the dyadic costs of the fixture, so run-to-run stable)."""
    code = (
        "import sys, os; sys.path.insert(0, %r); sys.argv = ['make_golden_mgm.py', 'mgm_ties', 'mgm_var_costs', 'mgm_max']\n"
        "import make_golden_mgm as m; m.G.GOLDEN = %r; m.main()\n") % (os.path.join(ROOT, "oracle"), str(tmp_path))
    subprocess.run([sys.executable, "-W", "ignore", "-c", code], check=True, capture_output=True, timeout=300)
    for name in ("mgm_ties", "mgm_var_costs", "mgm_max"):
        new = np.load(os.path.join(str(tmp_path), name + ".npz"))
        old = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        for k in ("value", "cost", "gain", "new_value", "cycle_count", "var_rank", "tables", "unary"):
            assert np.array_equal(new[k], old[k], equal_nan=True), (name, k)


@settings(max_examples=20, deadline=None)
@given(st.integers(4, 30), st.integers(2, 6), st.integers(2, 40), st.sampled_from([2, 3]),
       st.integers(0, 10_000))
def test_mgm_properties(n_vars, d, n_factors, arity, seed):
    """Per round no two neighbours move together, and with integer costs and fresh (non-stale)
    information the global cost never increases: MGM's monotonicity, which the restatement keeps
    in min mode as long as costs are exact."""
    arity = min(arity, n_vars)
    inst = random_factor_graph(n_vars, d, n_factors, arity, seed=seed, int_tables=True, noise=0.0)
    vp, ve = default_var_csr(n_vars, inst["edge_var"])
    inst = dict(inst, var_ptr=vp, var_edge=ve)
    o = orc.MgmOracle(inst, np.float64, mode="min", seed=seed).init()
    a = orc.MgmOracle(inst, np.float64, mode="min", seed=seed).init()
    assert np.array_equal(o.val, a.val)
    for _ in range(8):
        before = o.val.copy()
        o.step()
        moved = np.nonzero(o.val != before)[0]
        ms = set(moved.tolist())
        for v in moved:
            nb = set(o.nbr_idx[o.nbr_ptr[v]:o.nbr_ptr[v + 1]].tolist()) if o.has_nbr[v] else set()
            assert not (nb & ms), "two neighbours moved in the same round"
    a.step(8)
    assert np.array_equal(o.val, a.val)  # deterministic given the seed


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
def test_infinite_cost_fixtures_regenerate_bit_for_bit(tmp_path):
    code = (
        "import sys, os; sys.path.insert(0, %r); sys.argv = ['make_golden_extra.py']\n"
        "import make_golden_extra as m; m.G.GOLDEN = %r; m.main()\n") % (os.path.join(ROOT, "oracle"), str(tmp_path))
    subprocess.run([sys.executable, "-W", "ignore", "-c", code], check=True, capture_output=True, timeout=300)
    written = sorted(f[:-4] for f in os.listdir(str(tmp_path)) if f.endswith(".npz"))
    assert written == golden_names("msx_"), written
    for name in written:
        new = np.load(os.path.join(str(tmp_path), name + ".npz"))
        old = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        for k in ("r_state", "q_state", "r_sent", "q_sent", "value", "tables"):
            assert np.array_equal(new[k], old[k], equal_nan=True), (name, k)


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_equals_live_reference_on_random_cases(seed):
    """oracle/fuzz_vs_reference.py: random instances, parameters and cost scales (1e-6 .. 1e18) through the
    unmodified reference in lock-step and through the oracle — MaxSum messages / send decisions / values,
    DSA and MGM values and costs, every cycle."""
    import json
    r = subprocess.run([sys.executable, "-W", "ignore", os.path.join(ROOT, "oracle", "fuzz_vs_reference.py"),
                        "30", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert out["cases"] == 30 and out["failures"] == [], out["failures"]
