"""MixedDSA on the CPU: the oracle (tests/_mixeddsa_oracle.py) against the reference's own lock-step trajectories
(tests/golden/mixeddsa_*.npz, written by tools/make_golden_mixeddsa.py from the unmodified MixedDsaComputation of
pydcop/algorithms/mixeddsa.py), what each fixture exercises, and the live reference on random instances where it is
importable."""
import os

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _mixeddsa_oracle import (BRANCH_HARD, BRANCH_IDLE, BRANCH_NONE, BRANCH_SOFT, BRANCH_STUCK_HARD,
                              BRANCH_STUCK_SOFT, MOVED, MixedDsaOracle)
from conftest import GOLDEN_DIR, ROOT, golden_names

FIXTURES = golden_names("mixeddsa_")
# fixtures whose costs are integers or multiples of 1/8: every operation is exact in f32 as well
EXACT_F32 = [n for n in FIXTURES if n != "mixeddsa_ref_gc10"]


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def oracle_for(inst, meta, dt):
    return MixedDsaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"])


def check_trajectory(run, inst, meta, dt, name):
    """Compare `run` (init()/step()/values()/record()) with a fixture, round by round; f32 runs compare with the
    fixture's costs rounded to f32."""
    for k in range(meta["n_cycles"] + 1):
        if k:
            run.step()
        val, cost = run.values()
        assert np.array_equal(val, inst["value"][k]), (name, k, "value")
        known = ~np.isnan(inst["cost"][k])
        assert np.array_equal(~np.isnan(cost), known), (name, k, "has_cost")
        assert np.array_equal(cost[known].astype(dt), inst["cost"][k][known].astype(dt)), (name, k, "cost")
        if k:
            rec = run.record()
            for key in ("h_best", "branch"):
                assert np.array_equal(rec[key], inst[key][k]), (name, k, key)


def test_fixture_set():
    assert 14 <= len(FIXTURES) <= 16
    variants = {load(n)[1]["params"]["variant"] for n in FIXTURES}
    assert variants == {"A", "B", "C"}
    assert {load(n)[1]["mode"] for n in FIXTURES} == {"min", "max"}
    assert load("mixeddsa_rand_d12")[0]["dom_size"].max() == 12


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_f64_reproduces_reference_trajectory(name):
    inst, meta = load(name)
    check_trajectory(oracle_for(inst, meta, np.float64).init(), inst, meta, np.float64, name)


@pytest.mark.parametrize("name", EXACT_F32)
def test_oracle_f32_reproduces_exact_cost_fixtures(name):
    inst, meta = load(name)
    t = inst["tables"][np.isfinite(inst["tables"])]
    assert np.array_equal(t * 8, np.round(t * 8)) and np.array_equal(inst["unary"] * 8, np.round(inst["unary"] * 8))
    check_trajectory(oracle_for(inst, meta, np.float32).init(), inst, meta, np.float32, name)


def branches(name):
    b = load(name)[0]["branch"][1:]
    return b & 7, (b & MOVED) != 0


# the branch (and whether it moved) each fixture is made for
WANTED = {
    "mixeddsa_defaults": [BRANCH_HARD, BRANCH_SOFT, BRANCH_STUCK_SOFT],
    "mixeddsa_variant_A": [BRANCH_HARD, BRANCH_SOFT],
    "mixeddsa_proba_1": [BRANCH_HARD, BRANCH_SOFT, BRANCH_STUCK_HARD, BRANCH_STUCK_SOFT],
    "mixeddsa_max_inf": [BRANCH_HARD, BRANCH_SOFT],
    "mixeddsa_stalemate": [BRANCH_STUCK_HARD],
    "mixeddsa_ties": [BRANCH_STUCK_SOFT],
    "mixeddsa_rand_d12": [BRANCH_HARD, BRANCH_SOFT],
}


@pytest.mark.parametrize("name", sorted(WANTED))
def test_fixture_moves_through_its_branches(name):
    br, moved = branches(name)
    for want in WANTED[name]:
        assert (moved & (br == want)).any(), (name, want)


def test_variant_c_is_variant_b():
    """The variant-C branch of the reference sits after `elif delta_dcop == 0` and never runs."""
    b, c = load("mixeddsa_defaults")[0], load("mixeddsa_variant_C")[0]
    for key in ("value", "cost", "h_best", "branch"):
        assert np.array_equal(b[key], c[key], equal_nan=True), key
    a = load("mixeddsa_variant_A")[0]
    assert not np.array_equal(a["value"], b["value"])
    br, moved = branches("mixeddsa_variant_A")
    assert not (br == BRANCH_STUCK_SOFT).any()


def test_zero_probabilities_never_move():
    inst, _ = load("mixeddsa_proba_0")
    assert (inst["value"] == inst["value"][0]).all()
    assert np.isnan(inst["cost"]).all()
    br, moved = branches("mixeddsa_proba_0")
    assert not moved.any() and (br == BRANCH_HARD).any()


def test_infinite_entries():
    """+inf in max mode is still a violation; a -inf entry is a hard constraint whose cost is added, and a -inf
    current cost against a -inf best makes dC NaN: no move."""
    inst, meta = load("mixeddsa_max_inf")
    assert meta["mode"] == "max" and (inst["h_best"][1:] > 0).any() and np.isposinf(inst["tables"]).any()
    for name in ("mixeddsa_neg_inf_min", "mixeddsa_neg_inf_max"):
        inst, meta = load(name)
        assert np.isneginf(inst["tables"]).any() and not np.isposinf(inst["tables"]).any()
        o = oracle_for(inst, meta, np.float64).init()
        nan_dc = 0
        for _ in range(meta["n_cycles"]):
            for v in range(o.V):
                if o.nbrs[v]:
                    h, c, _ = o.best_values(v, o.val)
                    cc, hc = o.dcop_cost(v, o.val)
                    with np.errstate(invalid="ignore"):
                        nan_dc += hc == h and np.isnan(cc - c)
            o.step()
        assert nan_dc > 0, name


def test_isolated_variables_evaluate_once():
    """'uno' (a unary constraint only) and 'iso' (no constraint) evaluate in round 1 only; 'iso' has H = 0 and
    never moves."""
    for name in FIXTURES:
        inst, _ = load(name)
        names = list(inst["var_names"])
        for v in ("uno", "iso"):
            i = names.index(v)
            assert inst["branch"][1, i] != BRANCH_NONE and (inst["branch"][2:, i] == BRANCH_NONE).all(), (name, v)
            assert (inst["h_best"][2:, i] == -1).all()
        i = names.index("iso")
        assert inst["branch"][1, i] == BRANCH_IDLE and inst["h_best"][1, i] == 0


def test_fixture_shapes():
    inst, _ = load("mixeddsa_nary")
    ar = set(np.diff(inst["factor_ptr"]).tolist())
    assert {1, 2, 3, 4} <= ar
    inst, _ = load("mixeddsa_initial_values")
    assert (inst["init_value"] >= 0).any() and (inst["init_value"] < 0).any()
    inst, _ = load("mixeddsa_var_costs")
    assert len(set(inst["unary"].tolist())) > 2
    inst, _ = load("mixeddsa_ref_gc10")
    assert np.isfinite(inst["tables"]).all()


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
def test_live_reference_on_random_instances():
    """Where the reference is importable: the oracle against the unmodified MixedDsaComputation on a few hundred
    random mixed instances, every mode and variant."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_mixeddsa as M
    n = 0
    for seed in range(240):
        rng = np.random.default_rng(1000 + seed)
        mode = ("min", "max")[seed % 2]
        params = dict(variant="ABC"[seed % 3], proba_hard=float(rng.choice([0.0, 0.5, 1.0])),
                      proba_soft=float(rng.choice([0.0, 0.5, 1.0])))
        vs, cs = M.colouring(rng, n=int(rng.integers(3, 9)), dom=int(rng.integers(1, 4)),
                             n_edges=int(rng.integers(2, 10)), hard_share=float(rng.uniform()), levels=3,
                             arities=(2, 1, 3), neg_inf=bool(seed % 5 == 0), name="r")
        if seed % 4 == 0:
            vs, cs = M.with_costs(rng, vs, cs)
        vs, cs = M.with_extras(vs, cs)
        arr, meta = M.run_mixeddsa(vs, M.relations(cs), params, mode, 6, seed=seed)
        check_trajectory(oracle_for(arr, meta, np.float64).init(), arr, meta, np.float64, seed)
        n += 1
    assert n == 240
