"""GPU: the device-only binary kernels of DSA, A-DSA and MGM at every compiled domain size, on unions of problems with
a Philox key and (DSA, A-DSA) a parameter set per problem, against the CPU oracle of every problem alone, bit for bit
after every cycle.  The kernels are k_dsa_step_cached<T, D, PS> (active-row, PYDCOP_B200_DSA_CACHE=1),
k_dsa_step_bin<T, D, PS> (oriented-table, PYDCOP_B200_DSA_CACHE=0), k_mgm_gain_cached<T, D> (MGM's default value
phase) and k_mgm_gain_bin<T, D, U> (PYDCOP_B200_MGM_CACHE=0 with PYDCOP_B200_MGM_FAST=U).  The instances, the
parameters and what shows that they took effect are in tests/_binary_unions.py."""
import numpy as np
import pytest

import _binary_unions as bu

pytestmark = pytest.mark.gpu

N_CYCLES = 30


def _engine_state(kind, eng):
    """The engine's side of bu.oracle_state, canonical order."""
    if kind != "mgm":
        return (eng.values(),)
    return eng.values() + eng.gains()


def _run(kind, D, mixed, precision):
    """Steps the union one cycle at a time and compares every problem's slice with its oracle; returns the engine."""
    dcops, params, seeds = bu.case(kind, D, mixed)
    traj = bu.case_trajectories(kind, D, mixed, precision, N_CYCLES)
    bu.check_non_vacuous(kind, traj, mixed)
    eng, u = bu.union_engine(kind, dcops, params, seeds, precision)
    assert bool(eng._desc.dev_var_seed)                                  # per-problem keys reach the descriptor
    if kind != "mgm":
        assert bool(eng._desc.dev_var_pset) == mixed and eng._desc.n_psets == (len(u.psets) if mixed else 0)
    eng.init()
    for k in range(N_CYCLES + 1):
        if k:
            eng.step()
        got = _engine_state(kind, eng)
        for i in range(len(dcops)):
            a, b = u.var_start[i], u.var_start[i + 1]
            for x, y in zip(got, traj[i][k]):
                assert np.array_equal(x[a:b], y, equal_nan=True), \
                    f"problem {i} ({params[i] if params else 'mgm'}, seed {seeds[i]}) differs after cycle {k}"
    return eng


def _clear_knobs(monkeypatch):
    for name in ("PYDCOP_B200_NO_FAST", "PYDCOP_B200_DSA_CACHE", "PYDCOP_B200_MGM_FAST", "PYDCOP_B200_MGM_CACHE"):
        monkeypatch.delenv(name, raising=False)


def _dsa(kind, D, mixed, precision, cache, monkeypatch):
    _clear_knobs(monkeypatch)
    monkeypatch.setenv("PYDCOP_B200_DSA_CACHE", cache)     # read at every step (dsa_cached_step): set for the run
    eng = _run(kind, D, mixed, precision)
    assert eng.tables_or is not None and eng._desc.fast_dom == D     # the oriented-table arrays, not the generic path
    last = eng.slot_last.cpu().numpy()[:eng.layout.n_edges]
    if cache == "1":      # the active-row kernel read a row for every slot (isolated variables have none)
        assert (last != 255).all()
    else:                 # the active-row kernel never ran: k_dsa_step_bin did
        assert (last == 255).all()
    eng.close()


@pytest.mark.parametrize("mixed", [True, False], ids=["psets", "keys"])
@pytest.mark.parametrize("cache", ["1", "0"], ids=["cached", "bin"])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("D", bu.FAST_DOMS)
def test_dsa_binary_kernels_match_the_oracle(D, precision, cache, mixed, monkeypatch):
    _dsa("dsa", D, mixed, precision, cache, monkeypatch)


@pytest.mark.parametrize("cache", ["1", "0"], ids=["cached", "bin"])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 5, 10, 20])
def test_adsa_binary_kernels_match_the_oracle(D, precision, cache, monkeypatch):
    _dsa("adsa", D, True, precision, cache, monkeypatch)


@pytest.mark.parametrize("path", ["cached", "bin2", "bin4"])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("D", bu.MGM_DOMS)
def test_mgm_binary_value_phases_match_the_oracle(D, precision, path, monkeypatch):
    _clear_knobs(monkeypatch)
    chunk = 2 if path in ("cached", "bin2") else 4
    monkeypatch.setenv("PYDCOP_B200_MGM_FAST", str(chunk))        # both read when the engine is built
    monkeypatch.setenv("PYDCOP_B200_MGM_CACHE", "1" if path == "cached" else "0")
    eng = _run("mgm", D, False, precision)
    assert eng.fast_chunk == chunk and eng._desc.fast_dom == D and (eng.row_cache is not None) == (path == "cached")
    if path == "cached":
        assert (eng.slot_last.cpu().numpy()[:eng.layout.n_edges] != 255).all()
    eng.close()
