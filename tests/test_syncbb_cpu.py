"""SyncBB on the CPU: the oracle (tests/_syncbb_oracle.py) against the reference's own message traces
(tests/golden/syncbb_*.npz, written by tools/make_golden_syncbb.py from the unmodified pydcop/algorithms/syncbb.py),
what those fixtures exercise, and the oracle against the live reference on random instances where it is present."""
import itertools
import os
import sys

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _syncbb_oracle import TERMINATE, SyncbbOracle
from conftest import GOLDEN_DIR, ROOT, golden_names

FIXTURES = golden_names("syncbb_")
RUNNABLE = [n for n in FIXTURES if n not in ("syncbb_arity3", "syncbb_one_var")]
INTEGER = [n for n in RUNNABLE if "float" not in n]


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def oracle_for(inst, meta, dt=np.float64):
    return SyncbbOracle(inst, dt, meta["mode"], inst["var_rank"]).init()


def check_trace(o, inst, name):
    """Step by step: the message received, then every variable's bound and selection after it; at the end the
    final selection and the message and step counts."""
    n = int(inst["n_steps"])
    for k in range(n):
        kind, recv, plen, mub = o.message()
        assert (kind, recv, plen) == (int(inst["step_type"][k]), int(inst["step_recv"][k]),
                                      int(inst["step_plen"][k])), (name, k)
        want = inst["step_ub"][k]
        assert (np.isnan(want) and np.isnan(mub)) or mub == o.dt(want), (name, k, mub, want)
        assert o.step()
        assert np.array_equal(o.bounds(), inst["ub"][k].astype(o.dt)), (name, k)
        assert np.array_equal(o.values(), inst["sel"][k]), (name, k)
    assert o.finished and not o.step()
    assert o.steps == n and o.messages == int(inst["msg_count"])
    assert np.array_equal(o.values(), inst["final_sel"])
    assert np.array_equal(o.cycle_counts(), inst["cycle_count"])


@pytest.mark.parametrize("name", RUNNABLE)
def test_oracle_f64_reproduces_reference_trace(name):
    inst, meta = load(name)
    check_trace(oracle_for(inst, meta), inst, name)


@pytest.mark.parametrize("name", INTEGER)
def test_oracle_f32_reproduces_integer_traces(name):
    """Integer costs are exact in f32: the same trace, bound for bound."""
    inst, meta = load(name)
    check_trace(oracle_for(inst, meta, np.float32), inst, name)


def brute_force(inst, mode):
    fp, ev, toff = inst["factor_ptr"], inst["edge_var"], inst["table_off"]
    best = None
    for asg in itertools.product(*[range(int(d)) for d in inst["dom_size"]]):
        c = 0.0
        for f in range(len(fp) - 1):
            sc = ev[fp[f]:fp[f + 1]]
            idx = np.ravel_multi_index(tuple(asg[int(v)] for v in sc), tuple(int(inst["dom_size"][v]) for v in sc))
            c += float(inst["tables"][toff[f] + idx])
        if best is None or (c < best if mode == "min" else c > best):
            best = c
    return best


def assignment_cost(inst, sel):
    fp, ev, toff = inst["factor_ptr"], inst["edge_var"], inst["table_off"]
    c = 0.0
    for f in range(len(fp) - 1):
        sc = ev[fp[f]:fp[f + 1]]
        idx = np.ravel_multi_index(tuple(int(sel[v]) for v in sc), tuple(int(inst["dom_size"][v]) for v in sc))
        c += float(inst["tables"][toff[f] + idx])
    return c


def test_toy_problem_answers():
    """The reference unit test's asserted answers (test_algorithms_syncbb.py): all G in min mode, G R R G in max."""
    for name, want in (("syncbb_toy_min", [1, 1, 1, 1]), ("syncbb_toy_max", [1, 0, 0, 1])):
        inst, meta = load(name)
        assert list(inst["final_sel"]) == want
        assert list(oracle_for(inst, meta).run().values()) == want


def test_tutorial_cost_and_message_count():
    """graph_coloring_tuto.yaml: cost 12 with 23 messages, as the reference's docstring reports."""
    inst, meta = load("syncbb_tuto")
    o = oracle_for(inst, meta).run()
    assert assignment_cost(inst, o.values()) == 12 and o.messages == 23


def test_partial_cost_acceptance_misses_the_optimum():
    inst, meta = load("syncbb_partial_accept")
    o = oracle_for(inst, meta).run()
    assert o.stats["partial"] > 0
    assert assignment_cost(inst, o.values()) > brute_force(inst, "min") == meta["optimum"]


def test_max_mode_is_exhaustive():
    """Max mode prunes nothing: the last variable sees every full assignment, and the answer is the optimum."""
    for name in ("syncbb_toy_max", "syncbb_floats_max"):
        inst, meta = load(name)
        o = oracle_for(inst, meta).run()
        last = int(o.chain[-1])
        visits = int(((inst["step_recv"] == last) & (inst["step_type"] == 0)).sum())
        assert visits == int(np.prod(inst["dom_size"][o.chain[:-1]].astype(np.int64)))
        assert o.stats["rejected"] == 0 and o.stats["partial"] == 0
        assert assignment_cost(inst, o.values()) == brute_force(inst, "max")


def test_inf_entries_prune_even_at_an_infinite_bound():
    """`inf >= inf` prunes while the bound is still inf: candidates are rejected before any full assignment."""
    inst, meta = load("syncbb_inf")
    assert np.isinf(inst["tables"]).any()
    o = oracle_for(inst, meta).run()
    assert o.stats["pruned_by_inf"] > 0


def test_unary_constraints_and_variable_costs_are_ignored():
    """Dropping the unary constraints and the variable costs changes nothing in the trace."""
    inst, meta = load("syncbb_ignored")
    fp = inst["factor_ptr"]
    assert (np.diff(fp) == 1).any() and np.asarray(inst["unary"]).any()
    keep = [f for f in range(len(fp) - 1) if fp[f + 1] - fp[f] == 2]
    new = np.full(len(fp) - 1, -1)
    new[keep] = np.arange(len(keep))
    stripped = dict(dom_size=inst["dom_size"], edge_var=np.concatenate([inst["edge_var"][fp[f]:fp[f + 1]] for f in keep]),
                    factor_ptr=np.arange(0, 2 * len(keep) + 1, 2),
                    tables=np.concatenate([inst["tables"][inst["table_off"][f]:inst["table_off"][f + 1]] for f in keep]))
    vp, vc = inst["var_ptr"], inst["var_con"]
    cons = [[int(new[c]) for c in vc[vp[v]:vp[v + 1]] if new[c] >= 0] for v in range(len(vp) - 1)]
    stripped["var_ptr"] = np.concatenate([[0], np.cumsum([len(c) for c in cons])])
    stripped["var_con"] = np.array([c for cs in cons for c in cs], dtype=np.int64)
    stripped["table_off"] = np.concatenate([[0], np.cumsum([inst["table_off"][f + 1] - inst["table_off"][f]
                                                            for f in keep])])
    for k in ("var_rank", "cycle_count", "n_steps", "msg_count", "step_type", "step_recv", "step_plen", "step_ub", "ub", "sel", "final_sel"):
        stripped[k] = inst[k]
    check_trace(oracle_for(stripped, meta), stripped, "stripped")


def test_name_order_differs_from_canonical_order():
    inst, meta = load("syncbb_name_order")
    assert not np.array_equal(inst["var_rank"], np.arange(len(inst["var_rank"])))
    o = oracle_for(inst, meta)
    assert int(inst["step_recv"][0]) == int(o.chain[1]) != 1


def test_variable_without_constraints():
    inst, meta = load("syncbb_isolated")
    iso = [v for v in range(len(inst["dom_size"])) if inst["var_ptr"][v + 1] == inst["var_ptr"][v]]
    assert iso and (inst["final_sel"][iso] >= 0).all()


def test_infeasible_instance_selects_nothing():
    """Every full assignment costs inf: no bound ever improves, so no variable ever selects a value and every
    one finishes without one."""
    inst, meta = load("syncbb_infeasible")
    o = oracle_for(inst, meta).run()
    assert (o.values() == -1).all() and (inst["final_sel"] == -1).all() and inst["finished"].all()
    assert np.isinf(o.bounds()).all()


def test_arity3_is_refused():
    """The reference fails inside assignment_cost on the variable missing from the pair assignment; the oracle
    refuses such an instance up front and names the constraint."""
    inst, meta = load("syncbb_arity3")
    assert meta["error"].startswith("KeyError") and int(inst["n_steps"]) == 0
    with pytest.raises(ValueError, match="constraint 1 has arity 3"):
        SyncbbOracle(inst, np.float64, "min", inst["var_rank"])


def test_one_variable_is_refused():
    """With one variable the reference posts its start message to no computation (syncbb.py:210) and nothing else
    happens: no value, no termination.  The oracle refuses the instance."""
    inst, meta = load("syncbb_one_var")
    assert meta["dangling"] == 1 and int(inst["n_steps"]) == 0 and not inst["finished"].any()
    with pytest.raises(ValueError, match="at least two variables"):
        SyncbbOracle(inst, np.float64, "min").init()


def test_fixture_set_covers_the_quirks():
    shows = set()
    for name in FIXTURES:
        shows.update(load(name)[1]["shows"])
    assert {"toy_min", "toy_max", "tuto", "partial_accept", "non_dyadic", "inf_entries", "inf_prunes", "ignored",
            "name_order", "isolated", "infeasible", "error", "dangling", "exhaustive"} <= shows


def test_terminate_travels_down_the_chain():
    inst, meta = load("syncbb_tuto")
    o = oracle_for(inst, meta)
    tail = inst["step_type"][-(o.n - 1):]
    assert (tail == TERMINATE).all() and list(inst["step_recv"][-(o.n - 1):]) == list(o.chain[1:])


# ---- against the live reference ----------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


def _golden_driver():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_syncbb as M
    return M


@needs_ref
def test_oracle_matches_live_reference_on_random_instances():
    """A few hundred random small binary instances, both modes, shuffled names, mixed domains, inf entries."""
    M = _golden_driver()
    rng = np.random.default_rng(2026)
    levels = [np.arange(6.0), np.array([0.0, 0.5, 1.25, 3.0, np.inf]), np.array([0.1, 0.3, 0.7, 1.9])]
    for i in range(240):
        n = int(rng.integers(2, 7))
        sizes = [int(x) for x in rng.integers(1, 4, size=n)]
        n_edges = int(rng.integers(1, n * (n - 1) // 2 + 1))
        names = [f"v{int(x)}" for x in rng.permutation(n)]
        mode = "max" if i % 5 == 0 else "min"
        vs, cs = M.random_binary(int(rng.integers(1 << 30)), n, 0, n_edges, levels[i % 3], names=names,
                                 shuffle=bool(i % 2), dom_sizes=sizes)
        inst, meta = M.run_syncbb(vs, cs, mode)
        check_trace(SyncbbOracle(inst, np.float64, mode, inst["var_rank"]).init(), inst, f"random {i}")


@needs_ref
def test_regeneration_reproduces_committed_fixtures(tmp_path):
    """(The toy problem's scopes come from constraint_from_str, whose order follows string hashing.)"""
    M = _golden_driver()
    names = ["syncbb_tuto", "syncbb_inf", "syncbb_floats", "syncbb_arity3"]
    M.main(names, out_dir=str(tmp_path))
    for name in names:
        got, gm = orc.load_golden(str(tmp_path / (name + ".npz")))
        want, wm = load(name)
        assert gm["error"] == wm["error"]
        for k in want:
            assert np.array_equal(got[k], want[k], equal_nan=want[k].dtype.kind == "f"), (name, k)
